"""The baseline dictionaries on the host: the reference's pickles load, the per-class adapters of the forward-only plans
reproduce the reference's encode, the evaluation groups and list order, the errors, the engine's descriptor checks, and
the fp64 oracle (oracle/baselines_oracle.py) against the reference's own metrics (tests/golden/baselines.pt, written by
oracle/make_baselines_golden.py)."""
import ctypes as C
import io
import pickle

import pytest
import torch

import autoencoders.learned_dict as shim
from oracle import baselines_oracle as BO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ica import ICAEncoder
from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict, Rotation, TiedSAE, UntiedSAE
from sparse_coding_b200.topk_encoder import TopKLearnedDict

GOLDEN = BO.load_golden()
gaussian_rows, ica_from_golden, ica_rows = BO.gaussian_rows, BO.ica_from_golden, BO.ica_rows


def cases():
    return BO.golden_cases(GOLDEN)


# ---- pickles
def test_reference_pickles_load_as_the_shim_classes():
    for e in GOLDEN["random"]:
        rd = torch.load(io.BytesIO(e["pickle"]), weights_only=False)
        assert type(rd) is RandomDict and rd.n_feats == e["n"] and rd.activation_size == e["d"]
        assert torch.equal(rd.encoder, e["encoder"]) and torch.equal(rd.encoder_bias, torch.zeros(e["n"]))
        assert torch.equal(rd.get_learned_dict(), e["encoder"])              # raw rows, not normalised
    ir = torch.load(io.BytesIO(GOLDEN["identity_relu"][0]["pickle"]), weights_only=False)
    assert type(ir) is IdentityReLU and ir.n_feats == ir.activation_size == 32
    assert torch.equal(ir.bias, torch.zeros(32))


def test_pickled_names_are_the_references():
    assert shim.IdentityReLU is IdentityReLU and shim.RandomDict is RandomDict
    for obj in (IdentityReLU(16), RandomDict(16, 24)):
        raw = pickle.dumps(obj)
        assert b"autoencoders.learned_dict" in raw and type(obj).__name__.encode() in raw
        back = torch.load(io.BytesIO(_saved(obj)), weights_only=False)
        assert type(back) is type(obj)


def _saved(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    return buf.getvalue()


def test_reference_quirks():
    # IdentityReLU tests `if bias:`, which raises for a bias of more than one element
    with pytest.raises(RuntimeError) as e:
        IdentityReLU(32, torch.ones(32))
    assert f"RuntimeError: {e.value}" == GOLDEN["identity_relu_bias_error"]
    eye = IdentityReLU(8).get_learned_dict()
    assert eye.device.type == "cpu" and torch.equal(eye, torch.eye(8))
    # RandomDict draws from the global RNG at construction
    torch.manual_seed(5)
    rd = RandomDict(12, 20)
    torch.manual_seed(5)
    assert torch.equal(rd.encoder, torch.randn(20, 12))
    assert RandomDict(12).n_feats == 12


# ---- adapters
@pytest.mark.parametrize("e", GOLDEN["ica"], ids=lambda e: f"d{e['d']}")
def test_ica_adapter_matches_the_reference_encode(e):
    ica = ica_from_golden(e)
    x = ica_rows(e)[:64]
    enc, bias, dec, t = MT._sae_inputs(ica)
    assert enc.dtype == t.dtype == torch.float32 and torch.equal(bias, torch.zeros(e["d"]))
    code = (x.double() - t.double()) @ enc.double().T
    want = e["code"]
    assert torch.allclose(ica.encode(x), want, rtol=0, atol=1e-9 * float(want.abs().max()))
    # the adapter's matrices are the fp64 ones rounded to fp32: the error is that rounding, carried through the product
    scale = ((x.double() - t.double()).abs() + t.double().abs() * 2 ** -24) @ enc.double().abs().T
    assert float(((code - want).abs() / scale).max()) < 4 * 2 ** -24
    assert torch.equal(dec, ica.get_learned_dict())


def test_random_and_identity_adapters():
    torch.manual_seed(0)
    rd = RandomDict(16, 24)
    enc, bias, dec, t = MT._sae_inputs(rd)
    assert enc is rd.encoder and dec is rd.encoder and bias is rd.encoder_bias and t is None
    ir = IdentityReLU(16)
    enc, bias, dec, t = MT._sae_inputs(ir)
    assert torch.equal(enc, torch.eye(16)) and torch.equal(dec, torch.eye(16)) and bias is ir.bias and t is None
    x = torch.randn(40, 16)
    assert torch.equal(torch.clamp(x @ enc.T + bias, min=0.0), ir.encode(x))


# ---- grouping and order
def test_group_keys():
    torch.manual_seed(1)
    d = 32
    e = GOLDEN["ica"][0]
    lds = [TiedSAE(torch.randn(40, d), torch.zeros(40)), IdentityReLU(d), UntiedSAE(torch.randn(40, d), torch.randn(40, d),
                                                                                   torch.zeros(40)),
           RandomDict(d, 44), ica_from_golden(e), TopKLearnedDict(torch.randn(48, d), 3), RandomDict(d)]
    groups = MT._eval_groups(lds, True, 8)
    assert groups == {("tied", 40, d, False): [0], ("untied", 32, d, False): [1], ("untied", 40, d, False): [2],
                      ("random", 48, d, False): [3], ("ica", 32, d, False): [4], ("topk", 48, d, False): [5],
                      ("random", 32, d, False): [6]}
    # the existing kinds group as before without the baselines
    assert MT._eval_groups([lds[i] for i in (0, 2, 5)], True, 8) == {("tied", 40, d, False): [0],
                                                                     ("untied", 40, d, False): [1],
                                                                     ("topk", 48, d, False): [2]}
    for kind in ("random", "ica"):
        sig = _lib.SIGNATURES[kind]
        assert sig.variant == _lib.SCE_UNTIED and sig.decoder and not sig.centering
    assert _lib.SIGNATURES["random"].decoder_raw and not _lib.SIGNATURES["random"].code_linear
    assert _lib.SIGNATURES["ica"].code_linear and not _lib.SIGNATURES["ica"].decoder_raw


def test_list_order_negative_keys_and_empties():
    key = torch.tensor([[-3.0, -1.5, 7.0, -1e30, 0.0, -1.5]])
    frag = torch.tensor([[4, 9, -1, 2, -1, 1]])
    o = MT._list_order(key, frag)
    assert o.tolist() == [[5, 1, 0, 3, 2, 4]]           # -1.5 (frag 1), -1.5 (frag 9), -3, -1e30, then the empties
    ik = torch.tensor([[5, 0, 9, 3]])
    assert MT._list_order(ik, torch.tensor([[1, 2, -1, 0]])).tolist() == [[0, 3, 1, 2]]
    # non-negative keys: as before (empties last whatever their stored key)
    assert MT._list_order(torch.tensor([[0.0, 2.0, 5.0]]), torch.tensor([[3, -1, 1]])).tolist() == [[2, 0, 1]]


# ---- errors
def test_errors():
    e = GOLDEN["ica"][0]
    ica = ica_from_golden(e)
    ica.n_feats = 16
    with pytest.raises(ValueError, match="n_feats"):
        MT._eval_groups([ica], False, 8)
    with pytest.raises(ValueError, match="n_feats"):
        MT._eval_groups([ICAEncoder(32)], False, 8)                     # not fitted
    with pytest.raises(NotImplementedError, match="Rotation"):
        MT._eval_groups([Rotation(torch.eye(8))], False, 8)


def _desc(variant, **kw):
    base = dict(variant=variant, n_models=2, d=64, n=128, batch_max=256, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999,
                eps=1e-8, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-8)
    return _lib.SceDesc(**dict(base, **kw))


def test_descriptor_modifiers():
    lib = _lib.load()
    ws = lambda v: lib.sce_workspace_bytes(C.byref(_desc(v)))
    untied = ws(_lib.SCE_UNTIED)
    assert untied > 0
    for mod in (_lib.SCE_CODE_LINEAR, _lib.SCE_DECODER_RAW, _lib.SCE_CODE_LINEAR | _lib.SCE_DECODER_RAW):
        assert ws(_lib.SCE_UNTIED | mod) == untied                       # no workspace of their own
        dsc = _desc(_lib.SCE_UNTIED | mod)
        assert lib.sce_forward_stats_workspace_bytes(C.byref(dsc), 256) > 0
        assert lib.sce_fragments_workspace_bytes(C.byref(dsc), 256, 64) > 0
        for other in (_lib.SCE_TIED, _lib.SCE_TOPK, _lib.SCE_TIED_LEARNED_CENTER):
            assert ws(other | mod) == 0
    for bad in (1 << 10, 1 << 16, 3 << 8 | 1 << 11):
        assert ws(_lib.SCE_UNTIED | bad) == 0
    assert ws(4) == 0


# ---- the fp64 oracle against the reference's own metrics
@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_oracle_against_golden(case):
    name, ld, m, x, want = case
    seg, thr = GOLDEN["segment"], GOLDEN["threshold"]
    c = BO.encode(m, x)
    assert torch.allclose(c, ld.encode(x).double(), rtol=0, atol=1e-5 * float(c.abs().max()))
    # (the reference averages in fp32)
    assert torch.allclose(BO.mean_nonzero_activations(m, x), want["mean_nonzero_activations"], rtol=0, atol=1e-6)
    assert BO.batched_calc_feature_n_ever_active(m, x, seg, thr) == want["n_ever_active"]
    got = dict(zip(("times_active", "mean", "var", "skew", "kurtosis", "m4"), BO.calc_moments_streaming(m, x, seg)))
    assert torch.equal(got["times_active"], want["moments"]["times_active"])
    for k in ("mean", "var", "skew", "kurtosis", "m4"):
        ref = want["moments"][k]
        assert torch.allclose(got[k], ref, rtol=1e-4, atol=1e-6 * float(ref.abs().max())), (name, k)
    fvu = BO.fraction_variance_unexplained(m, x)
    if "fvu_error" in want:
        assert name.startswith("ica") and "expected scalar type" in want["fvu_error"] and bool(fvu.isnan())
    else:
        assert abs(float(fvu) - want["fvu"]) <= 1e-5 * abs(want["fvu"])


@pytest.mark.parametrize("kind", ["ica", "random"])
def test_oracle_record_selection_against_golden(kind):
    """The fp64 oracle's fragment maxima on the stored fragments round to the reference's fp16 table, and its top 20
    fragments per feature carry the reference's maxima in the reference's order."""
    e = next(e for e in GOLDEN[kind] if e["interp"] is not None)
    if kind == "ica":
        m = BO.ica(e["scaler_mean"], e["scaler_scale"], e["components"], e["ica_mean"])
    else:
        rd = torch.load(io.BytesIO(e["pickle"]), weights_only=False)
        m = BO.random_dict(rd.encoder, rd.encoder_bias)
    ref = e["interp"]
    c = BO.encode(m, ref["acts"].float())
    fm = c.view(-1, 64, c.shape[1]).amax(dim=1).T         # [n, G] fp64
    want = ref["maxes"].double().T
    assert bool(((fm.half().double() - want).abs() <= want.abs() * 2.0 ** -10 + 2.0 ** -24).all())
    top = fm.sort(dim=1, descending=True, stable=True).indices[:, :20]
    assert torch.equal(want.gather(1, top), want.gather(1, ref["head"]))
    assert not bool(ref["skipped"].any())
    if kind == "ica":
        assert bool((want < 0).all(dim=1).any())
