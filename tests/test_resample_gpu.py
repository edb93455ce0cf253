"""Dead-feature tracking and resampling on the GPU (sce_step_tracked / sce_resample) against the fp64 oracle of
oracle/resample_oracle.py, for every signature the engine trains (tied, untied, masked tied and untied, learned centre,
positive tied, top-k on the gather and on the dense decode path) under both arithmetics.

Row errors e_r are held per row to a bound derived from the per-element x_hat bar of oracle/tile_bounds.py: with
|x_hat - x_hat*| <= bar S (S the absolute-product scale of x_hat), |e_r - e_r*| <= mean_d bar S (2 |x_hat* - x| + bar S),
doubled, plus the fp32 rounding of the row sum. Lists must hold the oracle's top N by fp64 error except rows within
that bound of the N-th value; rows, serials and counts are exact."""
import importlib.util
import os

import pytest
import torch

from oracle import resample_oracle as RO
from oracle import tile_bounds as T

pytestmark = pytest.mark.gpu

_spec = importlib.util.spec_from_file_location(
    "tile_bounds_checks", os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_tile_bounds_gpu.py"))
TB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(TB)

SHAPE = (4, 400, 1040, 1000)          # M, d, n, B (B <= n: one step from an empty window lists every row)
VARIANTS = ["tied", "untied", "masked_tied", "masked_untied", "learned_center", "positive_tied", "topk_gather",
            "topk_dense"]
ORACLE_NAME = {"tied": "tied", "untied": "untied", "masked_tied": "masked_tied", "masked_untied": "masked_untied",
               "learned_center": "tied_learned_center", "positive_tied": "positive_tied", "topk_gather": "topk",
               "topk_dense": "topk"}
TOPK_K = {"topk_gather": (3, 8, 5, 8), "topk_dense": (16, 33, 17, 40)}


def arith_shape(variant, arith):
    return SHAPE   # (d and n are multiples of 16: f16f8 runs on it too)


def build(variant, arith, shape=SHAPE, seed=3):
    import sparse_coding_b200 as S
    M, d, n, B = shape
    if variant.startswith("topk"):
        torch.manual_seed(seed)
        ks = TOPK_K[variant][:M] if M <= 4 else [32] * M
        models, sig = [S.TopKEncoder.init(d, n, k) for k in ks], S.TopKEncoder
    else:
        models, sig = TB.make_models(variant, M, d, n, seed)
    return TB.ensemble(models, sig, arith), models


def main_key(ens):
    return ens._engine_sig.main


def snapshot(ens):
    c = lambda tree: {k: v.clone() for k, v in tree.items()}
    return c(ens.params), c(ens.optim_states["mu"]), c(ens.optim_states["nu"])


def xhat_bound(variant, arith, P, buf, X):
    """(e*, bound) per row of one model in fp64 on the device."""
    name = ORACLE_NAME[variant]
    code, e = RO.forward64(name, P, buf, X)
    p = {k: v.double() for k, v in P.items()}
    if name == "topk":
        W, _ = TB.O.unit_rows(p["dict"], floor=None)
        S_ = (X.double().abs() @ W.abs().T) * (code > 0) @ W.abs()
        bar = T.TOPK_BARS[arith]["x_hat"][1]
        xin = X.double()
    else:
        f = TB.oracle(variant, p, {k: v.double() if v.is_floating_point() else v for k, v in buf.items()}, X.double())
        W_dec = f["W"]
        S_ = T.x_hat_scale(f["Xabs"], f["W_enc"], p["encoder_bias"], W_dec)
        bar = T.BARS[arith][TB.sign(variant)]["x_hat"][1]
        xin = f["Xin"]
        code = f["c"]
    xh = code @ (W if name == "topk" else f["W"])
    dev = (xh - xin).abs()
    bound = 2 * (bar * S_ * (2 * dev + bar * S_)).mean(dim=-1) + 64 * 2.0 ** -24 * e
    return code, e, bound


def per_model(ens, m):
    P = {k: v[m] for k, v in ens.params.items()}
    buf = {k: v[m] for k, v in ens.buffers.items()}
    return P, buf


def data(shape, seed, scale=1.0):
    M, d, n, B = shape
    return TB.synth(B, d, seed) * scale


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_tracking_changes_nothing_and_row_errors(variant, arith):
    shape = arith_shape(variant, arith)
    M, d, n, B = shape
    a, _ = build(variant, arith, shape)
    b, _ = build(variant, arith, shape)
    b.track_dead_features()
    for step in range(3):
        X = data(shape, 10 + step)
        pre = snapshot(b)
        la, auxa = a.step_batch(X)
        lb, auxb = b.step_batch(X)
        for k in la:
            assert torch.equal(la[k], lb[k]), (step, k)
        assert torch.equal(auxa["c"].mean_nnz, auxb["c"].mean_nnz)
        if step == 0:
            # every row of the first step is listed (B <= n): each e_r against the oracle, their mean against the loss
            lists = b.worst_rows()
            for m in range(M):
                L = lists[m]
                assert L["err"].numel() == B
                order = torch.argsort(L["serial"])
                e = L["err"][order].double()
                assert torch.equal(L["serial"][order].cpu(), torch.arange(B))
                assert torch.equal(L["rows"][order], X)                       # bitwise copies of the rows fed
                rec = lb.get("l_reconstruction", lb["loss"])[m].double()
                assert abs(float(e.mean() - rec)) <= 1e-5 * float(rec), (m, float(e.mean()), float(rec))
                P = {k: v[m] for k, v in pre[0].items()}
                _, buf = per_model(b, m)
                _, e_ref, bound = xhat_bound(variant, arith, P, buf, X)
                ratio = ((e - e_ref).abs() / bound).max()
                if variant.startswith("topk"):   # rows whose k-th score ties are excluded by the support check below
                    ratio = ((e - e_ref).abs() / bound).quantile(0.99)
                assert float(ratio) <= 1.0, (m, float(ratio))
    for tree_a, tree_b in zip(snapshot(a), snapshot(b)):
        for k in tree_a:
            assert torch.equal(tree_a[k], tree_b[k]), k
    b.stop_tracking()                                    # without a window: the same launches as a plain step
    X = data(shape, 20)
    a.step_batch(X)
    b.step_batch(X)
    assert a.gpu_launches_last_call() == b.gpu_launches_last_call()


def _window(ens, shape, seeds, ragged=None):
    """Steps on `seeds` (the last batch ragged); returns the batches and the pre-step params of each."""
    M, d, n, B = shape
    batches, pres = [], []
    for i, s in enumerate(seeds):
        rows = ragged if (ragged and i == len(seeds) - 1) else B
        X = TB.synth(rows, d, s)
        pres.append(snapshot(ens)[0])
        ens.step_batch(X)
        batches.append(X)
    return batches, pres


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_window_lists_counts_and_resample(variant, arith):
    shape = arith_shape(variant, arith)
    M, d, n, B = shape
    N = 300
    ens, _ = build(variant, arith, shape, seed=5)
    if not variant.startswith("topk"):
        # features 0..63 dead by construction (bias -100), the rest clearly alive
        ens.params["encoder_bias"][:, :64] = -100.0
        ens.params["encoder_bias"][:, 64:] = 1.0
        ens.refresh()
    ens.track_dead_features(N)
    counts = torch.zeros(M, n, dtype=torch.int32, device="cuda")
    batches, pres = [], []
    for i, s in enumerate([21, 22, 23]):
        X = TB.synth(B if i < 2 else 333, d, s)
        pres.append(snapshot(ens)[0])
        ens.step_batch(X)
        ens.active_counts(X.shape[0], counts)
        batches.append(X)
    lists = ens.worst_rows()
    twin = [l["rows"].clone() for l in lists]
    allx = torch.cat(batches)
    for m in range(M):
        L = lists[m]
        assert torch.equal(L["counts"], counts[m])
        assert L["err"].numel() == N
        assert torch.equal(L["rows"], allx[L["serial"]])                  # rows and serials exact
        # oracle e over the window
        es, bs = [], []
        for X, P in zip(batches, pres):
            Pm = {k: v[m] for k, v in P.items()}
            _, buf = per_model(ens, m)
            _, e, bound = xhat_bound(variant, arith, Pm, buf, X)
            es.append(e)
            bs.append(bound)
        e, bound = torch.cat(es), torch.cat(bs)
        nth = torch.sort(e, descending=True).values[N - 1]
        want = set(torch.nonzero(e > nth + bound).flatten().tolist())
        allowed = set(torch.nonzero(e >= nth - bound).flatten().tolist())
        got = set(L["serial"].tolist())
        assert want <= got <= allowed, (m, len(want - got), len(got - allowed))
        if not variant.startswith("topk"):
            dead = (counts[m] == 0).nonzero().flatten()
            mask = ens.buffers.get("coef_mask")
            expect = torch.arange(64, device="cuda")
            if mask is not None:
                assert not bool(mask[m][:64].any())
            assert torch.equal(dead[dead < 64], expect) and bool((counts[m][64:][
                (mask[m][64:] == 0) if mask is not None else slice(None)] > 0).all())
    # resample
    key = main_key(ens)
    before = snapshot(ens)
    import sparse_coding_b200 as S
    health, amax, steps = ens.health(), ens.input_absmax(), S._lib.load().sce_get_step_count(ens._plan)
    res = ens.resample_dead_features(0.2)
    after = snapshot(ens)
    mask = ens.buffers.get("coef_mask")
    for m in range(M):
        dead = RO.dead_features(counts[m].cpu(), mask[m].cpu() if mask is not None else None)
        assert int(res["n_dead"][m]) == dead.numel()
        k = min(dead.numel(), N)
        assert int(res["n_replaced"][m]) == k
        rep = torch.nonzero(res["replaced"][m]).flatten().cpu()
        assert torch.equal(rep, dead[:k])
        o = RO.resample(before[0][key][m], twin[m].cpu(), dead, 0.2, mask[m] if mask is not None else None)
        got = after[0][key][m].cpu().double()
        rel = ((got[rep] - o["W"][rep]).abs() / o["W"][rep].abs().clamp(min=1e-30)).max() if k else 0.0
        assert float(rel) <= 2.0 ** -22, float(rel)
        keep = torch.ones(n, dtype=torch.bool)
        keep[rep] = False
        for name in before[0]:
            if name == key:
                assert torch.equal(after[0][name][m][keep.cuda()], before[0][name][m][keep.cuda()])
            else:
                assert torch.equal(after[0][name][m], before[0][name][m]), name
        for tree_b, tree_a in ((before[1], after[1]), (before[2], after[2])):
            for name in tree_b:
                if name in (key, "decoder"):
                    assert bool((tree_a[name][m][rep.cuda()] == 0).all())
                    assert torch.equal(tree_a[name][m][keep.cuda()], tree_b[name][m][keep.cuda()])
                elif name == "encoder_bias":
                    assert bool((tree_a[name][m][rep.cuda()] == 0).all())
                    assert torch.equal(tree_a[name][m][keep.cuda()], tree_b[name][m][keep.cuda()])
                else:
                    assert torch.equal(tree_a[name][m], tree_b[name][m]), name
    assert ens.health() == health and ens.input_absmax() == amax
    assert S._lib.load().sce_get_step_count(ens._plan) == steps
    assert ens._track["next_serial"] == 0 and int(ens._track["filled"].sum()) == 0
    assert int(ens._track["counts"].abs().sum()) == 0
    # planes: the next step equals that of an ensemble built afresh from the resampled state
    sd = ens.state_dict()
    clone = lambda tree: {k: (clone(v) if isinstance(v, dict) else v.clone()) for k, v in tree.items()}
    fresh = S.FunctionalEnsemble.from_state(dict(sd, params=clone(sd["params"]), buffers=clone(sd["buffers"]),
                                                 optim_states=clone(sd["optim_states"])))
    X = TB.synth(B, d, 77)
    la, _ = ens.step_batch(X)
    lb, _ = fresh.step_batch(X)
    for k in la:
        assert torch.equal(la[k], lb[k]), k
    for ta, tb in zip(snapshot(ens), snapshot(fresh)):
        for k in ta:
            assert torch.equal(ta[k], tb[k]), k


def test_repeatable_and_survives_rebuild_and_fallback():
    shape = (4, 400, 1040, 500)
    runs = []
    for _ in range(2):
        ens, _ = build("tied", "auto", shape, seed=9)
        ens.track_dead_features(200)
        ens.step_batch(TB.synth(500, 400, 1))
        ens.step_batch(TB.synth(900, 400, 2))                  # a larger batch: the plan is rebuilt, the window stays
        assert ens._plan_key[0] == 900
        runs.append([{k: v.clone() for k, v in l.items()} for l in ens.worst_rows()])
        assert ens._track["next_serial"] == 1400
    for a, b in zip(*runs):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert max(int(l["serial"].max()) for l in runs[0]) >= 500   # rows of the second batch entered
    # arith="auto": an out-of-range batch is skipped on f16f8 and re-run on bf16x3; it enters the window once
    ens, _ = build("tied", "auto", shape, seed=9)
    ens.track_dead_features(200)
    ens.step_batch(TB.synth(500, 400, 1))
    X = TB.synth(500, 400, 3)
    X[7, 3] = 1e5
    with pytest.warns(RuntimeWarning):
        ens.health_check_every = 1
        ens.step_batch(X)
    assert ens.resolved_arith() == "bf16x3"
    assert ens._track["next_serial"] == 1000
    for l in ens.worst_rows():
        s = l["serial"]
        assert s.unique().numel() == s.numel()
        assert 507 in s.tolist()                                 # the out-of-range row is the worst of its model
        assert torch.equal(l["rows"][(s >= 500).nonzero().flatten()], X[s[s >= 500] - 500])


@pytest.mark.parametrize("shape", [(16, 512, 4096, 8192), (1, 2048, 32768, 4096)], ids=["config2", "config5"])
def test_config_shapes_agree_with_the_oracle(shape):
    M, d, n, B = shape
    ens, _ = build("tied", "auto", shape, seed=11)
    N = n
    ens.track_dead_features()
    pres, batches = [], []
    for s in (31, 32):
        X = TB.synth(B, d, s)
        pres.append(snapshot(ens)[0])
        ens.step_batch(X)
        batches.append(X)
    arith = ens.resolved_arith()
    lists = ens.worst_rows()
    allx = torch.cat(batches)
    for m in range(M):
        L = lists[m]
        assert L["err"].numel() == min(N, 2 * B)
        assert torch.equal(L["rows"], allx[L["serial"]])
        es, bs = [], []
        for X, P in zip(batches, pres):
            Pm = {k: v[m] for k, v in P.items()}
            _, buf = per_model(ens, m)
            _, e, bound = xhat_bound("tied", arith, Pm, buf, X)
            es.append(e)
            bs.append(bound)
        e, bound = torch.cat(es), torch.cat(bs)
        if N < e.numel():
            nth = torch.sort(e, descending=True).values[N - 1]
            want = set(torch.nonzero(e > nth + bound).flatten().tolist())
            allowed = set(torch.nonzero(e >= nth - bound).flatten().tolist())
            got = set(L["serial"].tolist())
            assert want <= got <= allowed, (m, len(want - got), len(got - allowed))
        got_e = L["err"].double()
        ref = e[L["serial"]]
        assert bool(((got_e - ref).abs() <= bound[L["serial"]]).all())


def test_train_on_chunks_resamples_on_schedule(tmp_path):
    import numpy as np
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import train_on_chunks
    d, n_gt, bs = 128, 256, 512
    results = {}
    for mode in ("resample", "none", "zero"):
        np.random.seed(0)
        gen = S.SparseMixDataset(d, n_gt, 4096, 4, 1.0, 0.0, "cuda", sparse_component_covariance=torch.eye(n_gt),
                                 t_type=torch.float16, seed=7)
        torch.manual_seed(0)
        models = [S.FunctionalTiedSAE.init(d, 512, float(a)) for a in (1e-3, 3e-2)]
        ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
        chunks = S.SyntheticChunks(gen, 5, 4096)
        seen = []
        kw = {"resample": dict(resample_every=2, on_resample=lambda i, c, e, r: seen.append(
                  (i, r["n_dead"].tolist(), r["n_replaced"].tolist()))),
              "none": {}, "zero": dict(resample_every=0)}[mode]
        out = tmp_path / mode
        train_on_chunks(ens, {"device": "cuda"}, None, str(out), bs, [], ["l1_alpha"], chunks=chunks,
                        save_schedule="every", **kw)
        results[mode] = torch.load(out / "_4" / "learned_dicts.pt", weights_only=False)
        if mode == "resample":
            assert [s[0] for s in seen] == [0, 2, 4]
            for _, dead, rep in seen:
                assert rep == [min(x, 512) for x in dead]
            assert ens._track is None
    a, b = results["none"], results["zero"]
    for (da, ha), (db, hb) in zip(a, b):
        assert ha == hb
        for k, v in vars(da).items():
            if isinstance(v, torch.Tensor):
                assert torch.equal(v, vars(db)[k]), k
