"""Shared test code: the dense step's per-tile harness, the sparse-mixture batches, the dictionaries of the evaluation
tests and small helpers. Importing it needs no GPU; its functions that build tensors run on cuda:0.

The harness (make_models, ensemble, oracle, measure, check, run_case) checks every dense training-step output per
(model, 128 x 128 tile) and per element against fp64 with the bars of oracle/tile_bounds.py; tests/test_tile_bounds_gpu.py
states what it measures and how the bars were set."""
import torch

import sparse_coding_b200 as S
from oracle import learned_center_oracle as LC
from oracle import positive_tied_oracle as PT
from oracle import sae_oracle as O
from oracle import tile_bounds as T
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

DEV = torch.device("cuda", 0)
ARITHS = ["bf16x3", "f16f8"]
VARIANTS = ["tied", "tied_centering", "untied", "masked_tied", "masked_untied", "learned_center", "positive_tied"]
RAGGED = (4, 400, 1040, 4001)        # M, d, n, B
RAGGED_EAGER = (4, 400, 1040, 8001)  # the same, above the launch-bound rule (oracle/plan_paths.py)
NEAR_FRAC = 5e-4                     # bound on the share of coefficients inside the kink window
EXACT_ZERO_FLOOR = 3e-5              # bias-gradient error / scale above which an exact-zero pre-activation is looked for


# ---- small helpers
def relnorm(a, b):
    a, b = a.double(), b.double().to(a.device)
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def raw(t):
    """The bytes of a tensor, for bitwise comparison."""
    t = t.detach().contiguous().cpu()
    return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy().tobytes()


def clone_models(ms):
    return [({k: v.clone() for k, v in p.items()}, {k: v.clone() for k, v in b.items()}) for p, b in ms]


def desc(M, n, d, B, **fields):
    """An SceDesc of M models of n features, width d and batch_max B: a tied plan with three passes each way, Adam's
    defaults at lr 1e-3 and the norm floor 1e-8. ``fields`` sets any other field; the rest are 0."""
    base = dict(variant=_lib.SCE_TIED, x_per_model=0, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, eps_root=0.0,
                adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-8)
    return _lib.SceDesc(n_models=M, d=d, n=n, batch_max=B, **dict(base, **fields))


# ---- sparse-mixture batches
def synth(B, d, seed, fp16_values=True, n_feats=2048):
    """Sparse-mixture activations, generated on the device: each row a non-negative mix of about 1 % of n_feats unit
    directions plus noise; fp16_values rounds them to fp16 (returned as fp32)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn(n_feats, d, generator=gen, device=DEV)
    feats /= feats.norm(dim=-1, keepdim=True)
    codes = (torch.rand(B, n_feats, generator=gen, device=DEV) < 0.01).float() * \
        torch.rand(B, n_feats, generator=gen, device=DEV)
    x = codes @ feats + 0.05 * torch.randn(B, d, generator=gen, device=DEV)
    return x.half().float() if fp16_values else x


def batch(M, B, d, seed, per_model, fp16_values, n_feats=2048):
    if per_model:
        return torch.stack([synth(B, d, seed + 7919 * m, fp16_values, n_feats) for m in range(M)])
    return synth(B, d, seed, fp16_values, n_feats)


# ---- dictionaries of the evaluation tests (LearnedDicts on the device)
def tied(n, d, seed, centering=(None, None, None)):
    """A TiedSAE whose biases leave some features active on most rows, most on few, some positive on an all-zero row."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return S.TiedSAE(torch.randn(n, d, generator=g, device=DEV), 0.05 * torch.randn(n, generator=g, device=DEV) - 0.03,
                     centering=centering)


def untied(n, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    enc = torch.randn(n, d, generator=g, device=DEV) / d ** 0.5
    return S.UntiedSAE(enc, torch.randn(n, d, generator=g, device=DEV), 0.05 * torch.randn(n, generator=g, device=DEV) - 0.03)


def topk(n, d, k, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return S.TopKLearnedDict(torch.nn.functional.normalize(torch.randn(n, d, generator=g, device=DEV), dim=-1), k)


def one_key(lds, arith, centre=False):
    """The key evaluate_dicts groups ``lds`` under (the dictionaries must share one)."""
    groups = MT._eval_groups(lds, centre, 16 if arith == "f16f8" else 8)
    assert len(groups) == 1, groups
    return next(iter(groups))


def as_oracle(ld):
    """A dictionary of oracle/eval_oracle.py (fp64) from a LearnedDict."""
    g = lambda t: t.double().to(DEV)
    if isinstance(ld, S.TopKLearnedDict):
        return {"kind": "topk", "dict": g(ld.dict), "sparsity": int(ld.sparsity)}
    if isinstance(ld, S.UntiedSAE):
        return {"kind": "untied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias), "decoder": g(ld.decoder)}
    return {"kind": "tied", "encoder": g(ld.encoder), "encoder_bias": g(ld.encoder_bias),
            "center_trans": g(ld.center_trans), "center_rot": g(ld.center_rot), "center_scale": g(ld.center_scale)}


# ---- the dense step's per-tile harness
def sign(variant):
    return "nonneg" if variant == "positive_tied" else "signed"


def make_models(variant, M, d, n, seed):
    torch.manual_seed(seed)
    gen = torch.Generator().manual_seed(seed + 1)
    models = []
    for m, a in enumerate(torch.logspace(-4, -2, M).tolist()):
        size = [n, n - 57, n // 2 + 3, n // 5 + 1][m % 4]     # masked dictionary sizes, not multiples of 128
        if variant == "tied":
            sig = S.FunctionalTiedSAE
            p, b = sig.init(d, n, a)
        elif variant == "tied_centering":
            sig = S.FunctionalTiedSAE
            q, _ = torch.linalg.qr(torch.randn(d, d, generator=gen))
            p, b = sig.init(d, n, a, translation=0.3 * torch.randn(d, generator=gen), rotation=q.contiguous(),
                            scaling=0.5 + torch.rand(d, generator=gen))
        elif variant == "untied":
            sig = S.FunctionalSAE
            p, b = sig.init(d, n, a, bias_decay=0.01)
        elif variant == "masked_tied":
            sig = S.FunctionalMaskedTiedSAE
            p, b = sig.init(d, size, n, a)
        elif variant == "masked_untied":
            sig = S.FunctionalMaskedSAE
            p, b = sig.init(d, size, n, a)
        elif variant == "learned_center":
            sig = S.FunctionalTiedCenteredSAE
            p, b = sig.init(d, n, a, center=0.1 * torch.randn(d, generator=gen))
        else:
            sig = S.FunctionalPositiveTiedSAE
            p, b = sig.init(d, n, a, 0.01)
        if variant != "positive_tied":
            p["encoder_bias"] = 0.02 * torch.randn(n, generator=gen)
        models.append((p, b))
    return models, sig


def ensemble(models, sig, arith, **kw):
    return S.FunctionalEnsemble(clone_models(models), sig, S.adam, {"lr": 1e-3}, device="cuda", arith=arith, **kw)


def oracle(variant, P, buf, X, active=None):
    """fp64 forward of one model (and, given the activity pattern ``active``, its gradients), with the batch the loss
    sees (``Xin``: centred or shifted) and the encoder matrix the code is computed from (``W_enc``)."""
    alpha = float(buf["l1_alpha"])
    bd = float(buf["bias_decay"]) if "bias_decay" in buf and not variant.startswith("masked") else 0.0
    mask = buf["coef_mask"].bool() if variant.startswith("masked") else None
    E, b = P["encoder"], P["encoder_bias"]
    if variant in ("untied", "masked_untied"):
        Xin, W_enc = X, E
        f = (O.untied_forward(E, b, P["decoder"], X, alpha, bd, mask) if active is None else
             O.untied_grads(E, b, P["decoder"], X, alpha, bd, mask, active))
    elif variant == "learned_center":
        Xin = X - P["center"][None, :]
        f = O.tied_forward(E, b, Xin, alpha) if active is None else \
            LC.tied_center_grads(E, b, P["center"], X, alpha, active)
    elif variant == "positive_tied":
        Xin = X + PT.SHIFT
        f = O.tied_forward(E.clamp(min=0.0), b, Xin, alpha, bd) if active is None else \
            PT.positive_tied_grads(E, b, X, alpha, bd, active)
    else:
        Xin = X if variant != "tied_centering" else \
            O.center(X, buf["center_trans"].double(), buf["center_rot"].double(), buf["center_scale"].double())
        f = O.tied_forward(E, b, Xin, alpha, bd, mask) if active is None else \
            O.tied_grads(E, b, Xin, alpha, bd, mask, active)
    if variant not in ("untied", "masked_untied"):
        W_enc = f["W"]
    Xabs = Xin.abs() if variant != "tied_centering" else \
        T.centered_input_scale(X, buf["center_trans"].double(), buf["center_rot"].double(), buf["center_scale"].double())
    f.update(Xin=Xin, Xabs=Xabs, W_enc=W_enc, bd=bd, alpha_over_B=alpha / X.shape[0])
    if active is not None:
        f["gate"] = (active | (f["Z"] == 0)) & (~mask if mask is not None else True)
    return f


def scales(variant, f, b):
    """Absolute-product scale of every gradient the signature has (oracle/tile_bounds.py)."""
    S_dz = T.pre_activation_grad_scale(f["G"], f["W"], f["alpha_over_B"], f["gate"])
    out = {"encoder_bias": T.bias_grad_scale(S_dz, O._bias_decay_grad(b, f["bd"]))}
    if variant not in ("untied", "masked_untied"):
        out["encoder"] = T.row_norm_jacobian_scale(f["W"], f["s"], T.weight_grad_scale(S_dz, f["Xabs"], f["c"], f["G"]))
    else:
        out["encoder"] = T.weight_grad_scale(S_dz, f["Xabs"])
        out["decoder"] = T.row_norm_jacobian_scale(f["W"], f["s"], T.weight_grad_scale(None, None, f["c"], f["G"]))
    if variant == "learned_center":
        out["center"] = T.center_grad_scale(f["G"], out["encoder_bias"], f["W"])
    return out


def regate_exact_zeros(variant, f, db_engine, candidates):
    """A pre-activation the engine computes as exactly 0 is inactive in its code and mask but passes the reconstruction
    gradient, without the L1 term (clamp's gradient at 0); the API does not read that bit back, and the pinned oracle has
    the coefficient closed. A feature whose bias-gradient error is explained to 90 % by one candidate (inside the kink
    window, zero code) gets that coefficient opened in ``f``: dz = g w^T there, added to the bias, encoder (and centre)
    gradients. Only an error above EXACT_ZERO_FLOOR of the bias gradient's scale qualifies, so at most one coefficient's
    worth of error per feature is explained away, and the caller bounds how many are. Returns the coefficients opened."""
    G, W, X = f["G"], f["W"], f["Xin"]
    err = db_engine.double() - f["grads"]["encoder_bias"]
    floor = EXACT_ZERO_FLOOR * T.bias_grad_scale(T.pre_activation_grad_scale(G, W, f["alpha_over_B"], f["gate"]))
    opened = []
    for j in torch.nonzero(candidates.any(0) & (err.abs() > floor)).flatten().tolist():
        rows = torch.nonzero(candidates[:, j]).flatten()
        v = G[rows] @ W[j]
        k = int((err[j] - v).abs().argmin())
        if not float((err[j] - v[k]).abs()) <= 0.1 * abs(float(err[j])):
            continue
        r, dz = int(rows[k]), float(v[k])
        dw = dz * X[r]
        f["grads"]["encoder_bias"][j] += dz
        if variant in ("untied", "masked_untied"):
            f["grads"]["encoder"][j] += dw
        else:
            f["grads"]["encoder"][j] += (dw - W[j] * (W[j] @ dw)) / f["s"][j]
        if "center" in f["grads"]:
            f["grads"]["center"] -= dz * W[j]
        f["gate"][r, j] = True
        opened.append((r, j))
    return opened


def measure(variant, ens, X, per_model):
    """Engine outputs of one grads_batch / forward_batch on X against the fp64 oracle, every model, every tile.
    Returns (T.Worst, kink counts per model)."""
    grads, (loss, aux) = ens.grads_batch(X, expand_dims=not per_model)
    code = aux["c"].dense()
    counts = ens.active_counts(X.shape[-2])
    _, _, x_hat = ens.forward_batch(X, expand_dims=not per_model, return_x_hat=True)
    w, kinks = T.Worst(), []
    for m in range(ens.n_models):
        P = {k: v[m].double() for k, v in ens.params.items()}
        buf = {k: v[m] for k, v in ens.buffers.items()}
        Xm = (X[m] if per_model else X).double()
        f0 = oracle(variant, P, buf, Xm)
        Z = f0["Z"]
        near = Z.abs() < T.kink_window(Z)
        eng_pos = T.engine_activity(code[m], counts[m], near, Z)
        across = eng_pos != (f0["c"] > 0)                      # (a masked coefficient is 0 on both sides)
        kinks.append((int(near.sum()), int((across & near).sum()), int((across & ~near).sum()), Z.numel()))
        del across
        S_code = T.code_scale(f0["Xabs"], f0["W_enc"], P["encoder_bias"])
        w.add("code", m, T.tile_ratios(code[m], f0["c"], S_code))
        w.add("x_hat", m, T.tile_ratios(x_hat[m], f0["x_hat"], S_code @ f0["W"].abs()))
        del S_code
        want = {"l_reconstruction": f0["l_reconstruction"], "l_l1": f0["l_l1"], "l_bias_decay": f0["l_bias_decay"],
                "loss": f0["l_reconstruction"] + f0["l_l1"] + f0["l_bias_decay"]}
        for k in loss:
            v = float(want[k])
            w.add_scalar("loss", m, abs(float(loss[k][m]) - v) / abs(v) if v != 0 else abs(float(loss[k][m])))
        active = torch.where(near, eng_pos, Z > 0)
        f = oracle(variant, P, buf, Xm, active)
        closed = near & ~eng_pos & (code[m] == 0)
        if "coef_mask" in buf:
            closed &= ~buf["coef_mask"].bool()
        opened = regate_exact_zeros(variant, f, grads["encoder_bias"][m], closed)
        kinks[-1] += (len(opened),)
        del f0, Z, near, eng_pos
        for k, S_ in scales(variant, f, P["encoder_bias"]).items():
            w.add(k, m, T.tile_ratios(grads[k][m], f["grads"][k], S_))
        del f, active
    return w, kinks


def report(tag, arith, variant, w, kinks=None):
    for name in w.tile:
        ratio, where = w.tile[name]
        tb, eb = T.BARS[arith][sign(variant)][name]
        at = f"model {where[0]}" + (f" tile ({where[1]}, {where[2]})" if len(where) == 3 else "")
        print(f"{tag:44s} {arith:6s} {name:12s} worst tile {ratio:.2e} at {at:24s} element max {w.elem[name]:.2e} | "
              f"bars {tb:.1e} {eb:.1e} | smallest tile {w.minimum[name][0]:.2e} element {w.minimum[name][1]:.2e}")
    if kinks:
        print(f"{tag:44s} {arith:6s} kink window per model (inside, engine across inside, across outside, of, opened "
              f"at an exact zero): {kinks}")


def check(tag, variant, ens, X, per_model, arith):
    w, kinks = measure(variant, ens, X, per_model)
    report(tag, arith, variant, w, kinks)
    for name, (ratio, where) in w.tile.items():
        tb, eb = T.BARS[arith][sign(variant)][name]
        assert ratio <= tb, (tag, name, "tile", ratio, where, tb)
        assert w.elem[name] <= eb, (tag, name, "element", w.elem[name], eb)
    for m, (inside, across_in, across_out, total, opened) in enumerate(kinks):
        assert across_out == 0, (tag, m, "flipped outside the kink window", across_out)
        assert inside <= NEAR_FRAC * total, (tag, m, inside, total)
        assert opened <= 2 + 1e-7 * total, (tag, m, "coefficients at an exact zero", opened)
    return w


def run_case(tag, variant, models, sig, arith, shape, per_model, fp16_values, steps=3, seed=100, n_feats=2048):
    M, d, n, B = shape
    ens = ensemble(models, sig, arith)
    X = batch(M, B, d, seed, per_model, fp16_values, n_feats)
    check(f"{tag} init", variant, ens, X, per_model, arith)
    assert ens.resolved_arith() == arith
    for s in range(steps):
        ens.step_batch(batch(M, B, d, seed + 1 + s, per_model, fp16_values, n_feats), expand_dims=not per_model)
    check(f"{tag} step{steps}", variant, ens, batch(M, B, d, seed + 50, per_model, fp16_values, n_feats), per_model,
          arith)


def bitwise_reruns(models, sig, arith, shape, seeds):
    """Two runs of the same steps on fresh ensembles of ``models``: two step_batch calls on batches of seeds[0] and
    seeds[0] + 1, then grads_batch on seeds[1]. Asserts every loss, code, gradient and parameter of the two bitwise
    equal, and returns the launch count of each run's last call."""
    M, d, _, B = shape

    def run():
        ens = ensemble(models, sig, arith)
        out = []
        for s in range(2):
            loss, aux = ens.step_batch(batch(M, B, d, seeds[0] + s, False, True))
            out += [v.clone() for _, v in sorted(loss.items())] + [aux["c"].dense().clone()]
        grads, _ = ens.grads_batch(batch(M, B, d, seeds[1], False, True))
        out += [v.clone() for _, v in sorted(grads.items())] + [v.clone() for _, v in sorted(ens.params.items())]
        return out, ens.gpu_launches_last_call()

    (a, la), (b, lb) = run(), run()
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and x.dtype == y.dtype, i
        assert raw(x) == raw(y), (shape, arith, i)
    return la, lb
