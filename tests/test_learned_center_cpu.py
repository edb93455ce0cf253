"""FunctionalTiedCenteredSAE (a tied SAE on x - center with the centre trained) without a GPU: the oracle against the
reference's recorded results, seeded init, the exported dictionary and the C ABI's host-side checks."""
import ctypes as C
import functools
import os

import pytest
import torch

from engine_cases import desc
from oracle import learned_center_oracle as LC
from oracle import sae_oracle as O
from sparse_coding_b200 import _lib

CASES = ["three_models", "mean_offset", "f64", "zero_center"]


@pytest.fixture(scope="module")
def cases(golden):
    return golden("tied_learned_center")


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(cases, name):
    fx = cases[name]
    tol = 1e-10 if fx["batch"].dtype == torch.float64 else 1e-5
    M = fx["params"]["encoder"].shape[0]
    for i in range(M):
        p = {k: v[i].double() for k, v in fx["params"].items()}
        f = LC.tied_center_grads(p["encoder"], p["encoder_bias"], p["center"], fx["batch"].double(),
                                float(fx["buffers"]["l1_alpha"][i]))
        for k in ("loss", "l_reconstruction", "l_l1"):
            assert abs(float(f[k]) - float(fx["loss_data"][k][i])) <= tol * abs(float(fx["loss_data"][k][i])), (k, i)
        assert rel(f["c"], fx["c"][i]) <= tol
        for k in ("center", "encoder", "encoder_bias"):
            assert rel(f["grads"][k], fx["grads"][k][i]) <= tol, (name, i, k, rel(f["grads"][k], fx["grads"][k][i]))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ref_port_signature_matches_closed_form(cases, dtype):
    """The vmap(grad) restatement (RefPortEnsemble's loss) against the closed form."""
    fx = cases["three_models"]
    params = {k: v.to(dtype) for k, v in fx["params"].items()}
    buffers = {k: v.to(dtype) for k, v in fx["buffers"].items()}
    X = fx["batch"].to(dtype)
    g = torch.vmap(torch.func.grad(LC.sig_loss_tied_learned_center, has_aux=True))
    grads, (loss, _) = g(params, buffers, X.expand(3, *X.shape))
    tol = 1e-10 if dtype == torch.float64 else 1e-5
    for i in range(3):
        f = LC.tied_center_grads(params["encoder"][i].double(), params["encoder_bias"][i].double(),
                                params["center"][i].double(), X.double(), float(buffers["l1_alpha"][i]))
        for k in grads:
            assert rel(grads[k][i], f["grads"][k]) <= tol, (k, i)
        assert abs(float(loss["loss"][i]) - float(f["loss"])) <= tol * float(f["loss"])


def test_zero_center_equals_tied(cases):
    """With a zero centre the signature is FunctionalTiedSAE: the reference's two losses and gradients agree."""
    fx = cases["zero_center"]
    assert float(fx["params"]["center"].abs().max()) == 0.0
    for k in ("encoder", "encoder_bias"):
        assert torch.equal(fx["grads"][k], fx["tied_grads"][k])
    for k in ("loss", "l_reconstruction", "l_l1"):
        assert torch.equal(fx["loss_data"][k], fx["tied_loss_data"][k])


@pytest.mark.parametrize("name", CASES)
def test_seeded_init_is_bitwise_the_references(cases, name):
    import sparse_coding_b200 as S
    fx = cases[name]
    a = fx["init"]
    torch.manual_seed(a["seed"])
    models = [S.FunctionalTiedCenteredSAE.init(a["d"], a["n"], l1, center=c.clone(), dtype=a["dtype"])
              for l1, c in zip(a["l1"], a["centers"])]
    for i, (p, b) in enumerate(models):
        assert list(p) == ["center", "encoder", "encoder_bias"] and list(b) == ["l1_alpha"]
        for k, v in p.items():
            assert torch.equal(v, fx["params"][k][i]), (name, k, i)
        assert torch.equal(b["l1_alpha"], fx["buffers"]["l1_alpha"][i])
    torch.manual_seed(a["seed"])
    p, _ = S.FunctionalTiedCenteredSAE.init(a["d"], a["n"], a["l1"][0], dtype=a["dtype"])
    assert torch.equal(p["center"], torch.zeros(a["d"], dtype=a["dtype"]))
    assert torch.equal(p["encoder"], fx["params"]["encoder"][0])   # the default centre draws no random numbers


def test_learned_dict_export(cases):
    import autoencoders.sae_ensemble as AS
    from sparse_coding_b200.learned_dict import TiedSAE
    fx = cases["three_models"]
    X = fx["batch"]
    for i in range(3):
        p = {k: v[i] for k, v in fx["params"].items()}
        b = {k: v[i] for k, v in fx["buffers"].items()}
        ld = AS.FunctionalTiedCenteredSAE.to_learned_dict(p, b)
        assert isinstance(ld, TiedSAE) and ld.norm_encoder
        assert torch.equal(ld.center_trans, p["center"])
        assert torch.equal(ld.center_rot, torch.eye(32)) and torch.equal(ld.center_scale, torch.ones(32))
        # LearnedDict.predict = uncenter(decode(encode(center(x)))): the reference's x_hat_centered + center
        f = O.tied_forward(p["encoder"].double(), p["encoder_bias"].double(), X.double() - p["center"].double(),
                           float(b["l1_alpha"]))
        assert rel(ld.predict(X), f["x_hat"] + p["center"].double()) <= 1e-5
        assert torch.allclose(AS.FunctionalTiedCenteredSAE.center(p, X), X - p["center"])
        assert torch.allclose(AS.FunctionalTiedCenteredSAE.uncenter(p, X), X + p["center"])
        w, floor, rows = AS.FunctionalTiedCenteredSAE.learned_dict_stack(fx["params"], fx["buffers"])
        assert w is fx["params"]["encoder"] and floor == 1e-8 and rows is None


# two learned-centre models, n = 128, d = 64, batch_max = 100
learned_desc = functools.partial(desc, 2, 128, 64, 100, variant=_lib.SCE_TIED_LEARNED_CENTER)


@pytest.fixture
def lib(monkeypatch):
    monkeypatch.delenv("SCE_ARITH", raising=False)
    return _lib.load()


def test_workspace_sizes(lib):
    for xpm in (0, 1):
        learned = lib.sce_workspace_bytes(C.byref(learned_desc(x_per_model=xpm)))
        tied_per_model = lib.sce_workspace_bytes(C.byref(learned_desc(x_per_model=1, variant=_lib.SCE_TIED)))
        assert learned > tied_per_model > 0   # M centred batches plus the centre-gradient buffers
    assert lib.sce_workspace_bytes(C.byref(learned_desc(x_per_model=0))) == \
        lib.sce_workspace_bytes(C.byref(learned_desc(x_per_model=1)))
    assert lib.sce_workspace_bytes(C.byref(learned_desc(x_per_model=1, centering=1))) == 0
    assert lib.sce_workspace_bytes(C.byref(learned_desc(variant=4))) == 0
    assert lib.sce_forward_stats_workspace_bytes(C.byref(learned_desc()), 64) == 0
    assert lib.sce_fragments_workspace_bytes(C.byref(learned_desc()), 64, 32) == 0
    assert lib.sce_forward_stats_workspace_bytes(C.byref(learned_desc(variant=_lib.SCE_TIED)), 64) > 0
    assert lib.sce_fragments_workspace_bytes(C.byref(learned_desc(variant=_lib.SCE_TIED)), 64, 32) > 0


def _create(lib, desc, with_center=True):
    """sce_plan_create on fake but non-null addresses: every check it fails here runs before it touches a device."""
    fake = 1 << 40
    bufs = _lib.SceBuffers()
    for name in ("encoder", "encoder_bias", "encoder_m", "encoder_v", "bias_m", "bias_v", "l1_alpha"):
        setattr(bufs, name, fake)
    if with_center:
        bufs.center, bufs.center_m, bufs.center_v = fake, fake, fake
    bufs.workspace, bufs.workspace_bytes = fake, 1 << 40
    plan = C.c_void_p()
    rc = lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan))
    return rc, lib.sce_last_error().decode()


def test_plan_create_rejections(lib):
    rc, msg = _create(lib, learned_desc(), with_center=False)
    assert rc == -1 and "center" in msg
    rc, msg = _create(lib, learned_desc(x_per_model=1, centering=2))
    assert rc == -1 and "centering" in msg
    # positive control: with the centre buffers the checks pass, and creation stops at the device query (no GPU here)
    rc, msg = _create(lib, learned_desc())
    assert rc != -1 or "center" not in msg


def test_export_declared_and_exported(lib):
    assert "sce_read_center_grad" in _lib.EXPORTS
    assert hasattr(lib, "sce_read_center_grad")
    header = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "sce.h")).read()
    assert "int sce_read_center_grad(sce_plan* plan, float* d_center, void* stream);" in header
    assert "SCE_TIED_LEARNED_CENTER = 3" in header
    assert lib.sce_version() == 201
    assert [f for f, _ in _lib.SceBuffers._fields_][-3:] == ["center", "center_m", "center_v"]
    assert lib.sce_read_center_grad(None, None, None) == -1


def test_signature_table_maps_the_signature():
    sig = _lib.SIGNATURES["tied_learned_center"]
    assert sig.variant == _lib.SCE_TIED_LEARNED_CENTER
    assert sig.loss_keys == ("loss", "l_reconstruction", "l_l1")
