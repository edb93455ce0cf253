"""FunctionalPositiveTiedSAE (a tied SAE on max(E, 0), trained on x + 0.18 with bias decay) without a GPU: the oracle
against the reference's recorded results, including its straight-through encoder gradient, seeded init, the exported
dictionary and the C ABI's host-side checks."""
import ctypes as C
import functools
import pickle

import pytest
import torch

from engine_cases import desc
from oracle import positive_tied_oracle as PT
from sparse_coding_b200 import _lib

CASES = ["fresh", "signed_encoder", "f64", "ratio1"]
LOSS_KEYS = ("loss", "l_reconstruction", "l_l1", "l_bias_decay")


@pytest.fixture(scope="module")
def cases(golden):
    return golden("positive_tied")


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300))


def model(fx, i):
    return ({k: v[i] for k, v in fx["params"].items()}, {k: v[i] for k, v in fx["buffers"].items()})


def oracle(fx, i):
    p, b = model(fx, i)
    return PT.positive_tied_grads(p["encoder"].double(), p["encoder_bias"].double(), fx["batch"].double(),
                                  float(b["l1_alpha"]), float(b["bias_decay"]))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(cases, name):
    fx = cases[name]
    tol = 1e-10 if fx["batch"].dtype == torch.float64 else 1e-5
    for i in range(fx["params"]["encoder"].shape[0]):
        f = oracle(fx, i)
        for k in LOSS_KEYS:
            ref = float(fx["loss_data"][k][i])
            assert abs(float(f[k]) - ref) <= tol * abs(ref) + (1e-12 if ref == 0 else 0), (name, k, i)
        assert rel(f["c"], fx["c"][i]) <= tol, (name, i)
        for k in ("encoder", "encoder_bias"):
            assert rel(f["grads"][k], fx["grads"][k][i]) <= tol, (name, i, k, rel(f["grads"][k], fx["grads"][k][i]))


def test_cases_cover_the_quirks(cases):
    """The fixture exercises what it is meant to: active codes on shifted MLP-like data, bias decay on and off, signed
    encoder entries and a row without a positive entry, d = n."""
    fresh = cases["fresh"]
    X = fresh["batch"]
    assert -0.18 < float(X.min()) < -0.16 and torch.equal(X, X.half().float())
    assert torch.equal(fresh["params"]["encoder_bias"], torch.full_like(fresh["params"]["encoder_bias"], -1.0))
    assert fresh["buffers"]["bias_decay"].tolist() == pytest.approx([0.01, 0.0, 0.01])
    assert fresh["buffers"]["l1_alpha"].tolist() == pytest.approx([0.0, 1e-4, 1e-3])
    assert float(fresh["loss_data"]["l_bias_decay"].max()) > 0 and float(fresh["loss_data"]["l_bias_decay"].min()) == 0
    for name in CASES:
        c = cases[name]["c"]
        assert bool((c > 0).any()), name
        # both sides of the ReLU, except at d = n = 64, where a fresh init on shifted data leaves every code positive
        assert bool((c == 0).any()) or name == "ratio1", name
    E = cases["signed_encoder"]["params"]["encoder"]
    assert bool((E < 0).any()) and bool((E == 0).any())
    assert bool(((E <= 0).all(-1)).any())
    assert cases["f64"]["batch"].dtype == torch.float64
    assert cases["ratio1"]["params"]["encoder"].shape[1] == cases["ratio1"]["params"]["encoder"].shape[2]


def test_straight_through_encoder_gradient(cases):
    """P1: the reference's encoder gradient is dL/dE+ with no [E >= 0] mask, so negative entries get gradient. The
    masked form, which a careful port might write, is far off on this case."""
    fx = cases["signed_encoder"]
    for i in range(fx["params"]["encoder"].shape[0]):
        p, b = model(fx, i)
        g_ref = fx["grads"]["encoder"][i]
        neg = p["encoder"] < 0
        assert float(g_ref[neg].abs().max()) > 0
        masked = PT.masked_encoder_grad(p["encoder"].double(), p["encoder_bias"].double(), fx["batch"].double(),
                                        float(b["l1_alpha"]), float(b["bias_decay"]))
        assert rel(masked, g_ref) > 1e-2, i
        assert rel(oracle(fx, i)["grads"]["encoder"], g_ref) <= 1e-5


def test_row_without_positive_entry(cases):
    """P6: a row with no positive entry has E+ = 0, so W's row is 0 and the norm floor 1e-8 divides its gradient: the
    reference's gradient there is dW / 1e-8, unguarded."""
    fx = cases["signed_encoder"]
    for i in range(fx["params"]["encoder"].shape[0]):
        E = fx["params"]["encoder"][i]
        rows = torch.nonzero((E <= 0).all(-1)).flatten().tolist()
        assert rows == [3]
        f = oracle(fx, i)
        assert float(f["W"][3].abs().max()) == 0.0 and float(f["s"][3]) == pytest.approx(1e-8)
        dW = f["dZ"].T @ (fx["batch"].double() + PT.SHIFT) + f["c"].T @ f["G"]
        assert rel(fx["grads"]["encoder"][i][3], dW[3] / 1e-8) <= 1e-5
        assert float(fx["grads"]["encoder"][i][3].norm()) > 1e3


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ref_port_signature_matches_closed_form(cases, dtype):
    """The vmap(grad) restatement (RefPortEnsemble's loss) against the closed form, on the case with signed entries."""
    fx = cases["signed_encoder"]
    params = {k: v.to(dtype) for k, v in fx["params"].items()}
    buffers = {k: v.to(dtype) for k, v in fx["buffers"].items()}
    X = fx["batch"].to(dtype)
    M = params["encoder"].shape[0]
    g = torch.vmap(torch.func.grad(PT.sig_loss_positive_tied, has_aux=True))
    grads, (loss, _) = g(params, buffers, X.expand(M, *X.shape))
    tol = 1e-10 if dtype == torch.float64 else 1e-5
    for i in range(M):
        f = oracle(fx, i)
        for k in grads:
            assert rel(grads[k][i], f["grads"][k]) <= tol, (k, i)
        for k in LOSS_KEYS:
            assert abs(float(loss[k][i]) - float(f[k])) <= tol * float(f[k]), (k, i)
    assert torch.equal(params["encoder"], fx["params"]["encoder"].to(dtype))   # the caller's tensors are untouched


@pytest.mark.parametrize("name", CASES)
def test_seeded_init_is_bitwise_the_references(cases, name):
    import sparse_coding_b200 as S
    fx = cases[name]
    a = fx["init"]
    torch.manual_seed(a["seed"])
    models = [S.FunctionalPositiveTiedSAE.init(a["d"], a["n"], l1, bd, dtype=a["dtype"])
              for l1, bd in zip(a["l1"], a["bias_decay"])]
    for i, (p, b) in enumerate(models):
        assert list(p) == ["encoder", "encoder_bias"] and list(b) == ["l1_alpha", "bias_decay"]
        for k, v in p.items():
            assert torch.equal(v, fx["init_params"][k][i]), (name, k, i)
        for k, v in b.items():
            assert torch.equal(v, fx["buffers"][k][i]), (name, k, i)
    torch.manual_seed(a["seed"])
    p, b = S.FunctionalPositiveTiedSAE.init(a["d"], a["n"], 1e-3, dtype=a["dtype"])
    assert float(b["bias_decay"]) == 0.0 and torch.equal(p["encoder"], fx["init_params"]["encoder"][0])


@pytest.mark.parametrize("name", ["fresh", "signed_encoder"])
def test_learned_dict_export(cases, name):
    """P5: the export is the reference's TiedSAE of the RAW encoder (negative entries kept) and bias, with no clamp and
    no translation by the shift."""
    from autoencoders.mlp_tests import FunctionalPositiveTiedSAE
    from sparse_coding_b200.learned_dict import TiedSAE
    fx = cases[name]
    d = fx["params"]["encoder"].shape[2]
    for i in range(fx["params"]["encoder"].shape[0]):
        p, b = model(fx, i)
        ld = FunctionalPositiveTiedSAE.to_learned_dict(p, b)
        assert isinstance(ld, TiedSAE) and ld.norm_encoder
        assert ld.encoder is p["encoder"] and ld.encoder_bias is p["encoder_bias"]
        assert torch.equal(ld.center_trans, torch.zeros(d)) and torch.equal(ld.center_rot, torch.eye(d))
        assert torch.equal(ld.center_scale, torch.ones(d))
        blob = pickle.dumps(ld)
        assert b"autoencoders.learned_dict" in blob and b"TiedSAE" in blob
        back = pickle.loads(blob)
        assert type(back) is TiedSAE and torch.equal(back.encoder, p["encoder"])
    w, floor, rows = FunctionalPositiveTiedSAE.learned_dict_stack(fx["params"], fx["buffers"])
    assert w is fx["params"]["encoder"] and floor == 1e-8 and rows is None
    if name == "fresh":
        ex = fx["export"]
        ld = FunctionalPositiveTiedSAE.to_learned_dict(*model(fx, 0))
        assert ex["type"] == "autoencoders.learned_dict.TiedSAE" and ex["norm_encoder"]
        assert torch.equal(ld.encoder, ex["encoder"]) and torch.equal(ld.encoder_bias, ex["encoder_bias"])
        assert rel(ld.get_learned_dict(), ex["learned_dict"]) <= 1e-6
        assert rel(ld.encode(ld.center(fx["batch"])), ex["encode"]) <= 1e-6
        assert rel(ld.predict(fx["batch"]), ex["predict"]) <= 1e-6


def test_public_names_and_engine_record():
    import autoencoders.mlp_tests as MT
    import sparse_coding_b200 as S
    assert MT.FunctionalPositiveTiedSAE is S.FunctionalPositiveTiedSAE
    assert "FunctionalPositiveTiedSAE" in S.__all__
    assert S.FunctionalPositiveTiedSAE.__module__ == "autoencoders.mlp_tests"
    assert S.FunctionalPositiveTiedSAE.variant == "positive_tied"
    sig = _lib.SIGNATURES["positive_tied"]
    assert sig.variant == _lib.SCE_TIED
    assert sig.loss_keys == LOSS_KEYS
    assert sig.input_shift == PT.SHIFT == 0.18


def test_unsupported_signature_error_names_it():
    import sparse_coding_b200 as S

    class Other(S.DictSignature):
        pass

    with pytest.raises(NotImplementedError, match="FunctionalPositiveTiedSAE"):
        S.FunctionalEnsemble([({"encoder": torch.zeros(8, 8)}, {})], Other, S.adam, {"lr": 1e-3})


# two non-negative tied models on x + 0.18, n = 128, d = 64, batch_max = 100
positive_desc = functools.partial(desc, 2, 128, 64, 100, encoder_nonneg=1, input_shift=0.18)


@pytest.fixture
def lib(monkeypatch):
    monkeypatch.delenv("SCE_ARITH", raising=False)
    return _lib.load()


def test_desc_fields_appended():
    names = [f for f, _ in _lib.SceDesc._fields_]
    assert names[-3:] == ["centering", "encoder_nonneg", "input_shift"]


def test_workspace_sizes(lib):
    ws = lambda **kw: lib.sce_workspace_bytes(C.byref(positive_desc(**kw)))
    for xpm in (0, 1):
        xm = 2 if xpm else 1
        tied = ws(x_per_model=xpm, encoder_nonneg=0, input_shift=0.0)
        assert tied > 0
        assert ws(x_per_model=xpm, input_shift=0.0) == tied              # the clamp needs no workspace
        shifted = (xm * 100 * 64 * 4 + 1023) // 1024 * 1024             # x + shift, [xm, batch_max, d] fp32
        assert ws(x_per_model=xpm) == tied + shifted
        assert ws(x_per_model=xpm, encoder_nonneg=0) == tied + shifted


@pytest.mark.parametrize("variant", [_lib.SCE_UNTIED, _lib.SCE_TOPK, _lib.SCE_TIED_LEARNED_CENTER])
@pytest.mark.parametrize("fields", [(1, 0.0), (0, 0.18), (1, 0.18)])
def test_fields_rejected_on_other_variants(lib, variant, fields):
    nonneg, shift = fields
    ws = lambda **kw: lib.sce_workspace_bytes(C.byref(positive_desc(variant=variant, x_per_model=1, **kw)))
    assert ws(encoder_nonneg=0, input_shift=0.0) > 0   # positive control
    assert ws(encoder_nonneg=nonneg, input_shift=shift) == 0


def test_validate_rejections(lib):
    ws = lambda **kw: lib.sce_workspace_bytes(C.byref(positive_desc(**kw)))
    assert ws(x_per_model=1, centering=2, input_shift=0.0) > 0     # centring with the clamp alone is allowed
    # the shift is not combined with centring
    assert ws(x_per_model=1, centering=2) == 0 and ws(x_per_model=1, centering=1) == 0
    assert ws(encoder_nonneg=2) == 0
    assert ws(input_shift=float("inf")) == 0 and ws(input_shift=float("nan")) == 0


def test_forward_only_passes_refused(lib):
    for nonneg, shift in ((1, 0.0), (0, 0.18), (1, 0.18)):
        d = positive_desc(encoder_nonneg=nonneg, input_shift=shift)
        assert lib.sce_forward_stats_workspace_bytes(C.byref(d), 64) == 0
        assert lib.sce_fragments_workspace_bytes(C.byref(d), 64, 32) == 0
    plain = positive_desc(encoder_nonneg=0, input_shift=0.0)
    assert lib.sce_forward_stats_workspace_bytes(C.byref(plain), 64) > 0
    assert lib.sce_fragments_workspace_bytes(C.byref(plain), 64, 32) > 0


def _create(lib, desc, coef_mask=False):
    """sce_plan_create on fake but non-null addresses: every check it fails here runs before it touches a device. On a
    machine with an sm_90 device a descriptor that passes them all gives a plan (creation touches no device memory),
    which is destroyed here; its rc is then 0, and sce_last_error still holds an earlier call's message."""
    fake = 1 << 40
    bufs = _lib.SceBuffers()
    for name in ("encoder", "encoder_bias", "encoder_m", "encoder_v", "bias_m", "bias_v", "l1_alpha", "bias_decay"):
        setattr(bufs, name, fake)
    if coef_mask:
        bufs.coef_mask = fake
    bufs.workspace, bufs.workspace_bytes = fake, 1 << 40
    plan = C.c_void_p()
    rc = lib.sce_plan_create(C.byref(desc), C.byref(bufs), C.byref(plan))
    msg = lib.sce_last_error().decode()
    if rc == 0:
        lib.sce_plan_destroy(plan)
    return rc, msg


def test_plan_create_rejects_the_fields_with_coef_mask(lib):
    for nonneg, shift in ((1, 0.0), (0, 0.18), (1, 0.18)):
        rc, msg = _create(lib, positive_desc(encoder_nonneg=nonneg, input_shift=shift), coef_mask=True)
        assert rc == -1 and "coef_mask" in msg, msg
    # positive controls: the masked tied plan alone, and the fields without a mask, pass these checks: creation goes on
    # to the device query, which fails without an sm_90 device (SCE_ERR_NO_DEVICE) and succeeds with one (SCE_OK)
    for desc, mask in ((positive_desc(encoder_nonneg=0, input_shift=0.0), True), (positive_desc(), False)):
        rc, msg = _create(lib, desc, coef_mask=mask)
        assert rc != -1, (rc, msg)
