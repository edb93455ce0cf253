"""NMFEncoder without a GPU: the reference's own fits (tests/golden/nmf.pt, sklearn's NMF()) against the fp64
restatement in oracle/nmf_oracle.py, the argument checks and workspace queries of sce_nmf_project / sce_nmf_grams /
sce_nmf_cd_sweep, and pickling."""
import ctypes as C
import io
import pickle

import numpy as np
import pytest
import torch

from oracle import nmf_oracle as O
from sparse_coding_b200 import _lib


def fixture_rows(g, case):
    """(training rows, held-out batches) of fit ``case``, fp16."""
    c = dict(g["cases"][case])
    n, held = c["n"], g["held_rows"]
    x = O.nmf_rows(c.pop("d"), c.pop("n") + sum(held), c.pop("seed"), **c)
    return x[:n], (x[n:n + held[0]], x[n + held[0]:])


def shifted(x, shift):
    return (x.double() - shift).clamp(min=0)


@pytest.mark.parametrize("case", ["d16", "d32", "shift16", "rank12", "sep16"])
def test_oracle_matches_reference_fit(golden, case):
    g = golden("nmf")
    f = g["fits"][case]
    x, held = fixture_rows(g, case)
    assert f["shift"] == (float(x.min()) if case == "shift16" else 0.0)
    X = shifted(x, f["shift"])
    W0, H0 = O.nndsvda(X)
    if case == "rank12":   # NNDSVDA fills the components of the zero singular values with the average
        assert torch.all(H0[12:] == X.mean()) and torch.all(W0[:, 12:] == X.mean())
    # the first two iterations' sweeps from the same start
    W, Ht = W0.clone(), H0.T.contiguous().clone()
    v = []
    for it in range(2):
        v.append(O.sweep(W, Ht.T @ Ht, X @ Ht))
        assert (W[:64] - f["sweeps"][2 * it]).abs().max() <= 1e-9 * W.abs().max(), (case, it)
        v.append(O.sweep(Ht, W.T @ W, X.T @ W))
        assert (Ht - f["sweeps"][2 * it + 1]).abs().max() <= 1e-9 * Ht.abs().max(), (case, it)
    assert np.allclose(v, f["violations"][:4], rtol=1e-9)
    r = O.fit(X, max_iter=f["max_iter"])
    assert r["n_iter"] == f["n_iter"]
    assert (r["H"] - f["components"]).abs().max() <= 1e-6 * f["components"].abs().max()
    assert abs(r["err"] - f["err"]) <= 1e-7 * f["err"]
    assert torch.equal(f["topk_rows"], f["components"].float())
    for h, ref in zip(held, f["held"]):
        codes, n_iter = O.transform(shifted(h, f["shift"]), f["components"])
        assert n_iter == ref["n_iter"]
        assert (codes - ref["codes"]).abs().max() <= 1e-8 * ref["codes"].abs().max()


@pytest.mark.parametrize("name", ["d32_it1", "d32_it3"])
def test_oracle_matches_reference_stopped_fit(golden, name):
    g = golden("nmf")
    s = g["stopped"][name]
    x, _ = fixture_rows(g, "d32")
    r = O.fit(shifted(x, 0.0), max_iter=s["max_iter"])
    assert r["n_iter"] == s["n_iter"] == s["max_iter"]
    assert (r["H"] - s["components"]).abs().max() <= 1e-9 * s["components"].abs().max()
    assert abs(r["err"] - s["err"]) <= 1e-9 * s["err"]


def test_reference_quirks_recorded(golden):
    g = golden("nmf")
    assert g["fp32_failure"].startswith("TypeError: H should have the same dtype as X")
    assert g["fp32_components_dtype"] == "float32"
    for f in g["fits"].values():
        assert f["components"].dtype == torch.float64
        assert any(h["n_iter"] < 200 for h in f["held"])


# ---- ABI (argument checks are made before any CUDA call)
def test_workspace_queries():
    lib = _lib.load()
    assert lib.sce_nmf_project_workspace_bytes(512, 512, 500) > 0
    assert lib.sce_nmf_grams_workspace_bytes(512, 512, 500) > 0
    assert lib.sce_nmf_cd_sweep_workspace_bytes(512, 500) > 0
    for d, k, B in ((4, 8, 10), (12, 8, 10), (16, 4, 10), (16, 24, 10), (8200, 8, 10), (64, 64, 0), (64, 64, (1 << 21) + 1)):
        assert lib.sce_nmf_project_workspace_bytes(d, k, B) == 0, (d, k, B)
        assert lib.sce_nmf_grams_workspace_bytes(d, k, B) == 0, (d, k, B)
    for k, R in ((0, 10), (2049, 10), (16, 0)):
        assert lib.sce_nmf_cd_sweep_workspace_bytes(k, R) == 0, (k, R)


@pytest.mark.parametrize("d", [8, 64, 512, 2048])
def test_workspace_never_decreases_with_rows(d):
    lib = _lib.load()
    grid = sorted({1, 2, 63, 64, 65, 255, 256, 257, 2047, 2048, 2049, 4095, 64000, 65536, 65537, 1 << 20,
                   (1 << 21) - 1, 1 << 21})
    for k in sorted({8, d // 2 // 8 * 8 or 8, d}):
        for q in (lib.sce_nmf_project_workspace_bytes, lib.sce_nmf_grams_workspace_bytes):
            needs = [q(d, k, B) for B in grid]
            assert all(n > 0 for n in needs), (q, d, k)
            assert all(a <= b for a, b in zip(needs, needs[1:])), (q.__name__, d, k, needs)
    for k in (1, 16, d, min(2048, 4 * d)):
        needs = [lib.sce_nmf_cd_sweep_workspace_bytes(k, B) for B in grid]
        assert all(n > 0 for n in needs) and all(a <= b for a, b in zip(needs, needs[1:])), (k, needs)


def _fake(n=0):
    """Aligned fake device addresses: the checks reject the arguments before any memory is touched."""
    return C.c_void_p(0x10000 + 1024 * n)


def test_project_and_grams_argument_checks():
    lib = _lib.load()
    ws = lib.sce_nmf_project_workspace_bytes(64, 64, 100)
    x, sh, m, p, nrm, flag, w = (_fake(i) for i in range(7))

    def project(**kw):
        a = dict(x=x, half=1, B=100, d=64, shift=sh, m=m, k=64, arith=0, p=p, norms=nrm, ws=_fake(40), ws_bytes=ws)
        a.update(kw)
        rc = lib.sce_nmf_project(a["x"], a["half"], a["B"], a["d"], a["shift"], a["m"], a["k"], a["arith"], a["p"],
                                 a["norms"], flag, a["ws"], a["ws_bytes"], None)
        return rc, lib.sce_last_error().decode()

    def grams(**kw):
        a = dict(x=x, B=100, d=64, w=w, k=64, arith=0, wtw=p, wtv=nrm)
        a.update(kw)
        rc = lib.sce_nmf_grams(a["x"], 1, a["B"], a["d"], sh, a["w"], a["k"], a["arith"], a["wtw"], a["wtv"], flag,
                               _fake(40), 1 << 30, None)
        return rc, lib.sce_last_error().decode()

    assert "p is required" in project(p=None)[1]
    assert "m is required" in project(m=None)[1]
    assert "x and shift are required" in project(x=None)[1]
    assert "x_is_half" in project(half=2)[1]
    assert "B = 0" in project(B=0)[1]
    assert "multiple of 8 in [8, 8192]" in project(d=12)[1]
    assert "k (72) must be a multiple of 8 in [8, d = 64]" in project(k=72)[1]
    assert "unknown arith" in project(arith=7)[1]
    assert "F16F8 needs d (64) and n (24)" in project(k=24, arith=2)[1]
    assert "16-byte aligned" in project(m=C.c_void_p(0x10008))[1]
    assert "p must be 16-byte aligned" in project(p=C.c_void_p(0x10008))[1]
    assert "workspace too small" in project(ws_bytes=ws - 1)[1]
    assert "1024-byte aligned" in project(ws=C.c_void_p(0x10010))[1]
    assert "wtw and wtv are required" in grams(wtv=None)[1]
    assert "w is required" in grams(w=None)[1]
    assert "k (4)" in grams(k=4)[1]
    assert "wtw and wtv must be 16-byte aligned" in grams(wtw=C.c_void_p(0x10008))[1]
    for rc, _ in (project(p=None), grams(w=None)):
        assert rc != 0


def test_residual_argument_checks():
    lib = _lib.load()
    x, sh, w, h, out = (_fake(i) for i in range(5))
    ws = lib.sce_nmf_residual_workspace_bytes(64, 100)
    assert ws > 0 and lib.sce_nmf_residual_workspace_bytes(12, 100) == 0 and lib.sce_nmf_residual_workspace_bytes(64, 0) == 0

    def res(**kw):
        a = dict(w=w, k=64, h=h, out=out, ws_bytes=ws)
        a.update(kw)
        rc = lib.sce_nmf_residual(x, 1, 100, 64, sh, a["w"], a["k"], a["h"], a["out"], _fake(40), a["ws_bytes"], None)
        return rc, lib.sce_last_error().decode()

    assert "h and sum are required" in res(h=None)[1]
    assert "w is required" in res(w=None)[1]
    assert "k (72)" in res(k=72)[1]
    assert "h must be 16-byte aligned" in res(h=C.c_void_p(0x10008))[1]
    assert "workspace too small" in res(ws_bytes=ws - 1)[1]
    grid = [1, 63, 64, 65, 4095, 65536, 1 << 21]
    needs = [lib.sce_nmf_residual_workspace_bytes(512, B) for B in grid]
    assert all(a <= b for a, b in zip(needs, needs[1:]))


def test_cd_sweep_argument_checks():
    lib = _lib.load()
    w, g, l, v, n = (_fake(i) for i in range(5))
    ws = lib.sce_nmf_cd_sweep_workspace_bytes(64, 100)

    def sweep(**kw):
        a = dict(w=w, f64=0, R=100, k=64, g=g, l=l, sweeps=1, tol=1e-4, v=v, n=None, ws=_fake(40), ws_bytes=ws)
        a.update(kw)
        rc = lib.sce_nmf_cd_sweep(a["w"], a["f64"], a["R"], a["k"], a["g"], a["l"], a["sweeps"], C.c_double(a["tol"]),
                                  a["v"], a["n"], a["ws"], a["ws_bytes"], None)
        return rc, lib.sce_last_error().decode()

    assert "are required" in sweep(l=None)[1]
    assert "w_is_f64" in sweep(f64=2)[1]
    assert "R (0)" in sweep(R=0)[1]
    assert "k (2049) must be in [1, 2048]" in sweep(k=2049)[1]
    assert "max_sweeps (3) must be 1 without n_iter" in sweep(sweeps=3)[1]
    assert "max_sweeps (0)" in sweep(sweeps=0, n=n)[1]
    assert "tol must be finite" in sweep(tol=float("nan"))[1]
    assert "aligned to their elements" in sweep(f64=1, w=C.c_void_p(0x10004))[1]
    assert "workspace too small" in sweep(ws_bytes=ws - 1)[1]


# ---- pickling and module names
def test_pickle_and_module_names():
    from autoencoders.nmf import FittedNMF, NMFEncoder
    from sparse_coding_b200.topk_encoder import TopKLearnedDict
    assert NMFEncoder.__module__ == FittedNMF.__module__ == "autoencoders.nmf"
    enc = NMFEncoder(16, n_components=32, shift=0.5)
    assert (enc.activation_size, enc.n_feats, enc.shift, enc.nmf) == (16, 32, 0.5, None)
    comps = np.abs(np.random.default_rng(0).normal(size=(16, 16)))
    enc.nmf = FittedNMF(comps, 7, 1.5, 1e-4, 200)
    enc._cache = ("not pickled",)
    blob = io.BytesIO()
    torch.save(enc, blob)
    back = torch.load(io.BytesIO(blob.getvalue()), weights_only=False)
    assert type(back) is NMFEncoder and not hasattr(back, "_cache")
    f = back.nmf
    assert (f.n_components_, f.n_features_in_, f.n_iter_, f.reconstruction_err_, f.tol, f.max_iter) == \
        (16, 16, 7, 1.5, 1e-4, 200)
    assert np.array_equal(f.components_, comps) and f.components_.dtype == np.float64
    assert pickle.loads(pickle.dumps(f)).n_iter_ == 7
    ld = back.get_learned_dict()
    assert ld.dtype == torch.float32 and torch.equal(ld, torch.tensor(comps, dtype=torch.float32))
    tk = back.to_topk_dict(3)
    assert isinstance(tk, TopKLearnedDict) and torch.equal(tk.dict, ld) and tk.sparsity == 3


def test_reference_pickle_loads(golden):
    pytest.importorskip("sklearn")
    g = golden("nmf")
    from autoencoders.nmf import NMFEncoder
    enc = torch.load(io.BytesIO(g["fits"]["d16"]["pickle"]), weights_only=False)
    assert type(enc) is NMFEncoder
    assert np.array_equal(enc.nmf.components_, g["fits"]["d16"]["components"].numpy())
    assert (enc.nmf.max_iter, enc.nmf.tol) == (200, 1e-4)


def test_fit_without_gpu_raises():
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    from autoencoders.nmf import NMFEncoder
    x = torch.rand(64, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        NMFEncoder(16).fit(x)
    with pytest.raises(ValueError, match="at least d"):
        NMFEncoder(16).fit(x[:8])
