"""ICAEncoder without a GPU: the reference's own fits (tests/golden/ica.pt, sklearn's StandardScaler + FastICA) against
the fp64 restatement in oracle/ica_oracle.py, the argument checks and workspace query of sce_ica_pass, pickling, and the
loud error of a fit without a CUDA device."""
import ctypes as C
import io
import pickle

import numpy as np
import pytest
import torch

from oracle import ica_oracle as O
from sparse_coding_b200 import _lib

TOL = 1e-4


def fixture_rows(g, name):
    """(training rows, held-out rows) of fit ``name``, fp64."""
    f = g["fits"][name]
    if "x" in f:
        return f["x"], f["held"]
    rows, _ = O.mixed_sources(f["d"], f["n"] + g["held_rows"], f["data_seed"])
    return rows[:f["n"]], rows[f["n"]:]


def n_iter_pinned(lims, tol=TOL):
    """Whether the iteration count is decided far from tol: the stopping lim is >= 10x below it, the others well above."""
    return lims[-1] <= tol / 10 and all(l >= 3 * tol for l in lims[:-1])


def sign_align(a, b):
    """``a`` with each row's sign set to agree with the same row of ``b``."""
    return a * torch.sign((a * b).sum(dim=1, keepdim=True))


@pytest.mark.parametrize("name", ["laplace2", "laplace4", "mixed32", "mixed64"])
def test_oracle_matches_reference_fit(golden, name):
    g = golden("ica")
    f = g["fits"][name]
    x, held = fixture_rows(g, name)
    r = O.fit(x, f["w_init"], max_iter=f["max_iter"])
    sc = f["scaler"]
    assert torch.allclose(r["mean"], sc["mean"], rtol=1e-12, atol=1e-14)
    assert torch.allclose(r["var"], sc["var"], rtol=1e-10)
    assert torch.allclose(r["scale"], sc["scale"], rtol=1e-10)
    assert sc["n"] == x.shape[0]
    # whitening from the covariance equals sklearn's SVD of the standardised rows, signs included
    assert (r["K"] - f["ica"]["whitening"]).norm() <= 1e-8 * f["ica"]["whitening"].norm()
    assert f["ica"]["mean"].abs().max() < 1e-12
    # W after 1 and 3 iterations from the same w_init (over the exactly whitened rows)
    n = x.shape[0]
    m, _, scale = O.standardise(x)
    xc = x - m
    K, Kw, _ = O.whitening(xc.T @ xc / n, scale, n)
    X1 = Kw @ xc.T
    W = O.sym_decorrelation(f["w_init"])
    lims = []
    for it in (1, 2, 3):
        W, lim = O.update(W, X1)
        lims.append(lim)
        if f"W{it}" in f:
            assert (W - f[f"W{it}"]).norm() <= 1e-8 * W.norm(), it
    assert np.allclose(lims[:len(f["lims"])], f["lims"][:3], rtol=1e-6, atol=1e-12)
    # the converged fit
    comp = f["ica"]["components"]
    assert (r["components"] - comp).norm() <= 1e-6 * comp.norm()
    assert (r["mixing"] - f["ica"]["mixing"]).norm() <= 1e-6 * f["ica"]["mixing"].norm()
    assert (r["W"] - f["ica"]["unmixing"]).norm() <= 1e-6 * f["ica"]["unmixing"].norm()
    if n_iter_pinned(f["lims"]):
        assert r["n_iter"] == f["n_iter"]
    assert torch.allclose(r["sources"][:g["held_rows"]], f["train_sources_head"], rtol=1e-6, atol=1e-6)
    held_src = ((held - r["mean"]) / r["scale"]) @ r["components"].T
    assert torch.allclose(held_src, f["held_sources"], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", ["mixed32_it1", "mixed32_it3", "mixed64_it1", "mixed64_it3"])
def test_oracle_matches_reference_stopped_fit(golden, name):
    g = golden("ica")
    s = g["stopped"][name]
    f = g["fits"][s["base"]]
    x, _ = fixture_rows(g, s["base"])
    r = O.fit(x, f["w_init"], max_iter=s["max_iter"])
    assert r["n_iter"] == s["n_iter"] == s["max_iter"]
    assert np.allclose(r["lims"], s["lims"], rtol=1e-6)
    assert (r["components"] - s["components"]).norm() <= 1e-8 * s["components"].norm()
    assert (r["W"] - s["unmixing"]).norm() <= 1e-8 * s["unmixing"].norm()


def test_reference_topk_export_cannot_encode(golden):
    """The reference's to_topk_dict hands numpy components to TopKLearnedDict; its encode fails (recorded at
    generation), which is why this repository's export carries torch rows."""
    assert golden("ica")["topk_failure"] is not None


def test_workspace_query_rejects_invalid_arguments():
    lib = _lib.load()
    assert lib.sce_ica_pass_workspace_bytes(512, 512, 500) > 0
    for d, n, B in ((0, 8, 10), (12, 8, 10), (8200, 8, 10), (64, 0, 10), (64, 12, 10), (64, 72, 10), (64, 64, 0),
                    (64, 64, -3), (64, 64, (1 << 21) + 1)):
        assert lib.sce_ica_pass_workspace_bytes(d, n, B) == 0, (d, n, B)


def test_workspace_need_never_decreases_with_rows():
    from sparse_coding_b200._rowpass import call_rows
    lib = _lib.load()
    for d, n in ((8, 8), (512, 512), (512, 256), (2048, 2048)):
        top = call_rows(d)
        needs = [lib.sce_ica_pass_workspace_bytes(d, n, B) for B in range(1, top + 1, 7)] + \
                [lib.sce_ica_pass_workspace_bytes(d, n, top)]
        assert all(v > 0 for v in needs)
        assert all(a <= b for a, b in zip(needs, needs[1:])), (d, n)
    assert lib.sce_ica_pass_workspace_bytes(512, 512, 64000) <= lib.sce_ica_pass_workspace_bytes(512, 512, 65536)
    assert lib.sce_ica_pass_workspace_bytes(2048, 2048, 1 << 21) > lib.sce_ica_pass_workspace_bytes(2048, 2048, 1 << 16)


def test_abi_rejects_bad_arguments_without_device():
    lib = _lib.load()
    fake = C.c_void_p(1 << 20)                 # never dereferenced: every check runs before any CUDA call
    need = lib.sce_ica_pass_workspace_bytes(64, 64, 100)

    def call(x=fake, half=1, B=100, d=64, shift=fake, unmix=fake, n=64, alpha=1.0, arith=0, gs=fake, gx=fake, ws=fake,
             ws_bytes=need):
        return lib.sce_ica_pass(x, half, B, d, shift, unmix, n, C.c_float(alpha), arith, gs, gx, None, ws, ws_bytes,
                                None)

    cases = [
        (dict(x=None), b"required"), (dict(shift=None), b"required"), (dict(unmix=None), b"required"),
        (dict(gs=None), b"required"), (dict(gx=None), b"required"), (dict(half=2), b"x_is_half"),
        (dict(B=0), b"outside"), (dict(B=(1 << 21) + 1), b"outside"), (dict(d=60), b"multiple of 8"),
        (dict(d=8200), b"8192"), (dict(n=12), b"multiple of 8"), (dict(n=72), b"[8, d"), (dict(alpha=0.5), b"alpha"),
        (dict(alpha=2.5), b"alpha"), (dict(alpha=float("nan")), b"alpha"), (dict(arith=5), b"unknown arith"),
        (dict(d=72, n=72, arith=_lib.SCE_ARITH_F16F8), b"multiples of 16"),
        (dict(n=24, arith=_lib.SCE_ARITH_F16F8), b"multiples of 16"),
        (dict(x=C.c_void_p((1 << 20) + 8)), b"aligned"), (dict(unmix=C.c_void_p((1 << 20) + 8)), b"aligned"),
        (dict(gx=C.c_void_p((1 << 20) + 8)), b"aligned"), (dict(gs=C.c_void_p((1 << 20) + 4)), b"aligned"),
        (dict(ws_bytes=need - 1), b"workspace too small"), (dict(ws=C.c_void_p((1 << 20) + 512)), b"1024-byte"),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc in (-1, -3), (kw, rc)
        assert msg in lib.sce_last_error(), (kw, lib.sce_last_error())


def test_pickle_round_trip_and_module():
    from sparse_coding_b200.ica import FittedFastICA, FittedScaler, ICAEncoder
    from autoencoders.ica import ICAEncoder as I2
    assert I2 is ICAEncoder and ICAEncoder.__module__ == "autoencoders.ica"
    r = O.fit(torch.from_numpy(np.random.RandomState(5).laplace(size=(400, 8))), torch.randn(8, 8, dtype=torch.float64))
    ica = ICAEncoder(8)
    a = lambda t: t.numpy()
    ica.scaler = FittedScaler(a(r["mean"]), a(r["var"]), a(r["scale"]), 400)
    ica.ica = FittedFastICA(a(r["components"]), a(r["mixing"]), np.zeros(8), a(r["K"]), a(r["W"]), r["n_iter"])
    blob = io.BytesIO()
    torch.save(ica, blob)
    assert pickle.dumps(ica).count(b"autoencoders.ica") >= 1
    back = torch.load(io.BytesIO(blob.getvalue()), weights_only=False)
    assert type(back) is ICAEncoder and back.ica.n_iter_ == r["n_iter"]
    x = torch.randn(16, 8, dtype=torch.float64)
    assert torch.equal(back.encode(x), ica.encode(x))
    assert torch.allclose(ica.encode(x), ((x - r["mean"]) / r["scale"]) @ r["components"].T)
    with pytest.raises(NotImplementedError, match="np.clamp"):
        ica.to_nneg_dict()
    ld = ica.get_learned_dict()
    assert ld.dtype == torch.float32 and torch.allclose(ld.norm(dim=1), torch.ones(8))
    tk = ica.to_topk_dict(3)
    assert tk.dict.shape == (16, 8) and torch.equal(tk.dict[8:], -tk.dict[:8])


def test_reference_pickle_encodes_here(golden):
    """An ica.pt the reference saved (with sklearn objects inside) encodes through this repository's class."""
    pytest.importorskip("sklearn")
    from sparse_coding_b200.ica import ICAEncoder
    g = golden("ica")
    for name in ("laplace2", "laplace4", "mixed32"):
        f = g["fits"][name]
        _, held = fixture_rows(g, name)
        ica = torch.load(io.BytesIO(f["pickle"]), weights_only=False)
        assert type(ica) is ICAEncoder
        assert torch.allclose(ica.encode(held), f["held_sources"], rtol=1e-12, atol=1e-12), name


def test_ica_needs_a_cuda_device():
    from sparse_coding_b200.ica import ICAEncoder
    x = torch.randn(100, 8)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ICAEncoder(8, device="cpu").train(x)
    with pytest.raises(ValueError, match="multiples of 8"):
        ICAEncoder(4, device="cpu").train(torch.randn(100, 4))
