"""Every top-k (TopKEncoder) training-step output of the engine per (model, 128 x 128 tile) and per element against fp64.

The top-k step runs kernels of its own: the scores epilogue with chunk maxima, topk_select2_kernel (which clears the
previous call's list entries in the code and code-gradient planes), the gather decode topk_sparse_kernel per k class and
per 2, 4 or 8 slices of d from the fp32 copy of the normalised dictionary that the dictionary-row kernel rewrites after
Adam, topk_dz_scatter_kernel, and a weight gradient that widens its f16f8 8-bit tiles (plan_config never gives top-k
dw_native). Outside the gather path (n < 96 kmax, kmax > 256, or no slice count fits) decode and dcode are the dense
GEMMs. test_topk_exact_gpu.py compares all of them bitwise, but on inputs the engine computes exactly, where every
residual plane is zero; here the inputs are arbitrary and every output is measured per tile against its absolute-
product scale (oracle/tile_bounds.py: topk_scales), over the whole output of every model:

  code      tiles of [B, n]   against the fp64 scores on the engine's support, scale |x| |W|^T on the support
  x_hat     tiles of [B, d]   against c W, scale (that scale) |W|
  dict      tiles of [n, d]   against sae_oracle.topk_grads on the engine's support, scale through the row-norm Jacobian
  loss      one relative error per model

The support the oracle is pinned to is the engine's: the code read back, plus any f16f8 code below ~4e-9 that reads as 0
while the activity mask has it on (engine_activity). It is checked separately to be the positive part of a top-k of the
fp64 scores up to the kink window (topk_support_check): no row keeps more than k, no kept score lies below a dropped one
by more than the window, outside the window the engine and fp64 keep the same columns, and the rows whose support
differs from fp64's own top-k at all are counted and bounded. Each case runs under both arithmetics with fp16-exact and
with fp32 inputs (whose residual plane is non-zero), at initialisation and again after 3 Adam steps on the engine's own
fp32 parameters as read back (the re-split planes, the fp32 dictionary copy of the gather path and, in launch-bound
plans, the graph-replayed step). Each case's path (gather launches, slices, graph) follows from the plan rule
(oracle/plan_paths.py) and is pinned by the launch count of every call. A call sequence on one plan (grads, a smaller
forward, grads on a new batch) checks the last call, where an entry of a residual plane left by an earlier call would
show.

Bars (tile ratio, element maximum; oracle/tile_bounds.py: TOPK_BARS) per arithmetic and output, set from measurement on
an H100 SXM (80 GB HBM3, 700 W limit): each is twice the worst 3-pass value this file observes at any case, rounded up.
The 1-pass column is the smallest non-empty tile of the single-pass runs (both ragged cases, fp32 inputs; fwd_passes=1
for code / x_hat, bwd_passes=1 for dict). Where it is at least twice the bar, the output is SEPARATED and
test_single_pass_tiles_clear_the_bars holds every such tile to it.

  arith   output  3-pass worst tile   bar      element max   bar      1-pass smallest tile   separated
  bf16x3  code    2.1e-6              4.3e-6   3.9e-6        7.8e-6   5.7e-5                 yes
          x_hat   3.3e-7              6.6e-7   2.5e-6        5.1e-6   7.4e-5                 yes
          dict    4.3e-7              8.7e-7   2.1e-5        4.2e-5   2.6e-5                 yes
  f16f8   code    7.8e-6              1.6e-5   1.6e-5        3.2e-5   5.3e-6                 no
          x_hat   1.4e-6              2.8e-6   9.2e-6        1.9e-5   9.3e-6                 yes (3.3x)
          dict    1.9e-6              3.9e-6   1.0e-4        2.1e-4   3.3e-6                 no

Losses (relative error per model): 3.0e-6 bf16x3, 1.3e-6 f16f8 (bars 6.1e-6, 2.6e-6); a 1-pass loss can be as exact,
so no loss is separated. The f16f8 code and dict gradient do not separate: their 3-pass error, fp32 rounding of scores
whose fp16 leading planes already carry 11 bits, is as large as the part a single pass drops (the same holds for the
dense variants' f16f8 gradients in tests/test_tile_bounds_gpu.py). Their bars still bound every tile and element at
twice the worst value measured. The rows whose support differs from fp64's own top-k at all, each inside the window,
reach 4.3e-3 of the batch (bound 9e-3); none differs outside it.

The x_hat error follows the code's: at 1 pass the gather path's x_hat (an fp32 sum over fp32 rows) has its smallest
tile at 7.4e-5 against 8.5e-5 for the dense decode at the same shape and 5.7e-5 for the code, and at 3 passes the
gather and dense x_hat worst tiles at the ragged shape are 3.3e-7 and 3.2e-7 (bf16x3), 1.2e-6 and 1.4e-6 (f16f8): the
decode's own rounding adds little. The whole file runs in about 30 s on an H100.
"""
import pytest
import torch

from engine_cases import batch, clone_models, synth
from oracle import sae_oracle as O
from oracle import tile_bounds as T
from oracle.plan_paths import gather_classes, gather_slices, launch_bound, launches

pytestmark = pytest.mark.gpu

ARITHS = ["bf16x3", "f16f8"]
REL = 1e-4                  # the per-model norm-relative bar of the other top-k parity tests
DIFFER_FRAC = 9e-3          # bound on the share of rows whose support differs from fp64's own top-k
BARS, SEPARATED = T.TOPK_BARS, T.TOPK_SEPARATED

CASES = {
    # id: (d, n, B, ks, gather launches, slices, graph-replayed step)
    # kmax = 8: the gather path with 2 slices; 33 chunks of 32 columns: selection on chunk maxima
    "ragged-gather-graph": (400, 1040, 4001, (3, 8, 5, 8), 1, 2, True),
    # kmax = 40 needs n >= 3840: the dense decode; k = 33, 40 exceed 32 per full warp: whole-row selection
    "ragged-dense-graph": (400, 1040, 4001, (16, 33, 17, 40), 0, 0, True),
    # every k class (<= 16, <= 32, <= 64, <= kmax = 104), n not a multiple of 128
    "every-k-class-eager": (400, 10000, 4001, (7, 16, 32, 33, 64, 100), 4, 2, False),
    # wide rows: kmax = 40 fits 4 slices of 512 columns, kmax = 64 needs 8
    "wide-4-slices": (2048, 6160, 2085, (16, 40), 2, 4, False),
    "wide-8-slices": (2048, 6160, 2085, (32, 64), 2, 8, False),
    # BASELINE config 3 at full size
    "cfg3-n6144": (768, 6144, 8192, (16, 32, 64), 3, 2, False),
    "cfg3-n12288": (768, 12288, 8192, (16, 32, 64), 3, 2, False),
}


def make_models(d, n, ks, seed):
    import sparse_coding_b200 as S
    torch.manual_seed(seed)
    return [S.TopKEncoder.init(d, n, k) for k in ks]


def ensemble(models, arith, **kw):
    import sparse_coding_b200 as S
    return S.FunctionalEnsemble(clone_models(models), S.TopKEncoder, S.adam, {"lr": 1e-3}, device="cuda", arith=arith,
                                no_stacking=True, **kw)


def path(cid):
    """The path of a case from the plan rule, checked against the case table."""
    d, n, B, ks, classes, slices, graph = CASES[cid]
    kr = (max(ks) + 7) // 8 * 8
    assert gather_classes(d, n, ks) == classes, (cid, gather_classes(d, n, ks))
    assert (gather_slices(d, kr) if classes else 0) == slices, (cid, gather_slices(d, kr))
    assert launch_bound(len(ks), B, n, d) == graph, cid
    return classes


def describe(cid):
    d, n, B, ks, classes, slices, graph = CASES[cid]
    return (f"{cid}: d {d} n {n} B {B} k {ks}: " + (f"gather, {classes} classes, {slices} slices" if classes else
            "dense decode") + f", step {'graph' if graph else 'eager'}, dw_native no")


def pinned_oracle(D, X, k, code, counts):
    """fp64 forward and gradients of one model on the engine's support, their scales and the support's check."""
    f0 = O.topk_forward(D, X, k)
    Z = f0["Z"]
    win = T.kink_window(Z)
    support = T.engine_activity(code, counts, Z.abs() < win, Z)
    sel = T.topk_support_check(Z, support, k, win)
    del f0
    f = O.topk_grads(D, X, k, support=support)
    # a kept score that fp64 puts at or below 0 (inside the window, where topk_support_check allows it) is positive in
    # the engine's fp32 scores, which pass its gradient
    edge = support & (f["Z"] <= 0)
    sel["edge"] = int(edge.sum())
    if sel["edge"]:
        f["dZ"] = f["dZ"] + (f["G"] @ f["W"].T) * edge.to(X.dtype)
        f["grads"]["dict"] = O._row_norm_jacobian(f["W"], f["s"], f["dZ"].T @ X + f["c"].T @ f["G"])
    scales = T.topk_scales(X, f["W"], f["s"], f["c"], f["G"], support)
    return f, scales, sel


def outputs(ens, X, per_model, classes, arith):
    """grads_batch, then forward_batch with x_hat, on X; the launch count of each call pinned to the case's path."""
    xm = X.shape[0] if per_model else 1
    grads, (loss, aux) = ens.grads_batch(X, expand_dims=not per_model)
    assert ens.gpu_launches_last_call() == launches("grads", classes, xm, arith)
    code = aux["c"].dense()
    counts = ens.active_counts(X.shape[-2])
    _, _, x_hat = ens.forward_batch(X, expand_dims=not per_model, return_x_hat=True)
    assert ens.gpu_launches_last_call() == launches("forward", classes, xm, arith)
    assert ens.resolved_arith() == arith
    return grads["dict"], loss["loss"], code, counts, x_hat


def nonempty(r):
    """tile_ratios' result with the tiles of zero error (the code's tiles without a kept entry, where both sides are
    0) left out of the smallest tile and element."""
    empty = r["ratio"] == 0
    inf = torch.full_like(r["ratio"], float("inf"))
    return dict(r, ratio=torch.where(empty, inf, r["ratio"]), peak=torch.where(empty, inf, r["peak"]))


def measure(ens, X, ks, per_model, classes, arith):
    """Every model's outputs against the fp64 oracle on its pinned support: (T.Worst, support checks per model)."""
    dW, loss, code, counts, x_hat = outputs(ens, X, per_model, classes, arith)
    w, sels = T.Worst(), []
    for m, k in enumerate(ks):
        D = ens.params["dict"][m].double()
        Xm = (X[m] if per_model else X).double()
        f, S, sel = pinned_oracle(D, Xm, k, code[m], counts[m])
        sels.append(sel)
        w.add("code", m, nonempty(T.tile_ratios(code[m], f["c"], S["code"])))
        w.add("x_hat", m, nonempty(T.tile_ratios(x_hat[m], f["x_hat"], S["x_hat"])))
        w.add("dict", m, nonempty(T.tile_ratios(dW[m], f["grads"]["dict"], S["dict"])))
        w.add_scalar("loss", m, abs(float(loss[m]) - float(f["loss"])) / float(f["loss"]))
        del f, S
    return w, sels


def report(tag, arith, w, sels=None):
    for name in w.tile:
        ratio, where = w.tile[name]
        tb, eb = BARS[arith][name]
        at = f"model {where[0]}" + (f" tile ({where[1]}, {where[2]})" if len(where) == 3 else "")
        print(f"{tag:40s} {arith:6s} {name:5s} worst tile {ratio:.2e} at {at:24s} element max {w.elem[name]:.2e} | "
              f"bars {tb:.1e} {eb:.1e} | smallest tile {w.minimum[name][0]:.2e} element {w.minimum[name][1]:.2e}")
    if sels:
        print(f"{tag:40s} {arith:6s} support per model (over k, misranked, rows differing, outside window, kept at "
              f"fp64 <= 0): {[tuple(s.values()) for s in sels]}")


def check(tag, ens, X, ks, per_model, classes, arith):
    w, sels = measure(ens, X, ks, per_model, classes, arith)
    report(tag, arith, w, sels)
    for name, (ratio, where) in w.tile.items():
        tb, eb = BARS[arith][name]
        assert ratio <= tb, (tag, name, "tile", ratio, where, tb)
        assert w.elem[name] <= eb, (tag, name, "element", w.elem[name], eb)
    B = X.shape[-2]
    for m, s in enumerate(sels):
        assert s["over_k"] == 0 and s["misranked"] == 0 and s["outside"] == 0, (tag, m, s)
        assert s["differ"] <= DIFFER_FRAC * B, (tag, m, s)
    return w


def run_case(cid, arith, fp16_values, per_model=False, steps=3, seed=100):
    d, n, B, ks, *_ = CASES[cid]
    classes = path(cid)
    M = len(ks)
    ens = ensemble(make_models(d, n, ks, 0), arith)
    tag = f"{cid} {'per-model' if per_model else 'shared'} {'fp16' if fp16_values else 'fp32'}"
    print(describe(cid))
    check(f"{tag} init", ens, batch(M, B, d, seed, per_model, fp16_values), ks, per_model, classes, arith)
    for s in range(steps):
        ens.step_batch(batch(M, B, d, seed + 1 + s, per_model, fp16_values), expand_dims=not per_model)
        assert ens.gpu_launches_last_call() == launches("step", classes, M if per_model else 1, arith)
    check(f"{tag} step{steps}", ens, batch(M, B, d, seed + 50, per_model, fp16_values), ks, per_model, classes,
          arith)


@pytest.mark.parametrize("inputs", ["fp16", "fp32"])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("cid", list(CASES))
def test_case_every_tile(cid, arith, inputs):
    run_case(cid, arith, inputs == "fp16")


@pytest.mark.parametrize("inputs", ["fp16", "fp32"])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("cid", ["ragged-gather-graph", "every-k-class-eager"])
def test_per_model_batches_every_tile(cid, arith, inputs):
    """expand_dims=False: every model reads its own batch (the gather kernel's per-model x stride)."""
    run_case(cid, arith, inputs == "fp16", per_model=True)


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("cid", ["ragged-gather-graph", "ragged-dense-graph"])
def test_call_sequence_last_call(cid, arith):
    """grads(B = 4001), forward(B = 1500), grads(B = 4001) on a new batch, arbitrary fp32 inputs, on one plan: the last
    call is checked per tile. An entry of a code or code-gradient residual plane that an earlier call left behind (a
    column it selected that this call does not) would show as an error in that row's code or dict-gradient tile."""
    d, n, B, ks, *_ = CASES[cid]
    classes = path(cid)
    ens = ensemble(make_models(d, n, ks, 1), arith)
    ens.grads_batch(synth(B, d, 700, False))
    ens.forward_batch(synth(1500, d, 701, False))
    print(describe(cid))
    check(f"{cid} sequence", ens, synth(B, d, 702, False), ks, False, classes, arith)


def single_pass(cid, arith, seed=500):
    """fwd_passes=1 (code, x_hat, loss) and bwd_passes=1 (the dict gradient) on a ragged case, fp32 inputs: what every
    tile of an output that lost its cross terms measures."""
    d, n, B, ks, *_ = CASES[cid]
    classes = path(cid)
    models = make_models(d, n, ks, 0)
    X = synth(B, d, seed, False)
    fwd, _ = measure(ensemble(models, arith, fwd_passes=1), X, ks, False, classes, arith)
    bwd, _ = measure(ensemble(models, arith, bwd_passes=1), X, ks, False, classes, arith)
    for attr in ("tile", "elem", "minimum"):
        getattr(fwd, attr)["dict"] = getattr(bwd, attr)["dict"]
    return fwd


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("cid", ["ragged-gather-graph", "ragged-dense-graph"])
def test_single_pass_tiles_clear_the_bars(cid, arith):
    """Every tile of a single-pass output measures at least twice its bar, for each output the bar separates."""
    w = single_pass(cid, arith)
    report(f"1-pass {cid}", arith, w)
    for name in SEPARATED[arith]:
        assert w.minimum[name][0] >= 2 * BARS[arith][name][0], (name, w.minimum[name][0], BARS[arith][name][0])


def _splice_last_tile(dst, src):
    """dst with its last (ragged) tile replaced by src's."""
    out = dst.clone()
    r0, c0 = (dst.shape[0] - 1) // 128 * 128, (dst.shape[1] - 1) // 128 * 128
    out[r0:, c0:] = src[r0:, c0:]
    return out


@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_single_pass_tile(arith):
    """The last, ragged tile of the last model's x_hat (from a fwd_passes=1 plan) and of its dict gradient (from a
    bwd_passes=1 plan) spliced into the 3-pass outputs of the gather case: the per-model norm-relative 1e-4 accepts each
    spliced tensor, the per-tile check rejects it at that tile, for each output whose bar separates 3-pass from 1-pass
    tiles; the numbers of the others are printed."""
    cid = "ragged-gather-graph"
    d, n, B, ks, *_ = CASES[cid]
    classes = path(cid)
    models = make_models(d, n, ks, 0)
    X = synth(B, d, 600, False)
    full = ensemble(models, arith)
    dW, _, code, counts, x_hat = outputs(full, X, False, classes, arith)
    _, _, x_hat1 = ensemble(models, arith, fwd_passes=1).forward_batch(X, return_x_hat=True)
    g1, _ = ensemble(models, arith, bwd_passes=1).grads_batch(X)
    m = len(ks) - 1
    f, S, _ = pinned_oracle(full.params["dict"][m].double(), X.double(), ks[m], code[m], counts[m])
    last = lambda t: ((t.shape[0] - 1) // 128, (t.shape[1] - 1) // 128)
    results = []
    for name, got, got1, want in (("x_hat", x_hat[m], x_hat1[m], f["x_hat"]),
                                  ("dict", dW[m], g1["dict"][m], f["grads"]["dict"])):
        spliced = _splice_last_tile(got, got1)
        rel = float((spliced.double() - want).norm() / want.norm())
        rel3 = float((got.double() - want).norm() / want.norm())
        r = T.tile_ratios(spliced, want, S[name])
        tile_bar = BARS[arith][name][0]
        print(f"negative control {arith:6s} {name:5s} spliced tile {last(want)}: norm-relative {rel:.2e} (3-pass "
              f"{rel3:.2e}, bar {REL:.0e}); worst tile {r['worst'][0]:.2e} at {r['worst'][1]}, tile bar {tile_bar:.1e}")
        results.append((name, rel, r["worst"], tile_bar, (0,) + last(want)))
    for name, rel, worst, tile_bar, at in results:
        if name not in SEPARATED[arith]:
            continue                       # no gap between 3-pass and 1-pass tiles of this output: no claim
        assert rel <= REL, (name, rel, REL)                                 # the per-model norm misses the tile ...
        assert worst[0] > tile_bar and worst[1] == at, (name, worst, at)    # ... the per-tile check does not
