"""BatchedPCA without a GPU: the reference's own fit (tests/golden/pca.pt) against the fp64 restatement in
oracle/pca_oracle.py, the reference's pickled exports loading into this repository's classes, the argument checks of
sce_second_moments, and the loud error of a BatchedPCA without a CUDA device."""
import ctypes as C
import io
import pickle

import pytest
import torch

from oracle import pca_oracle as O
from sparse_coding_b200 import _lib


def test_oracle_matches_reference_fit(golden):
    g = golden("pca")
    x = g["x"].double()
    mean, cov = O.moments(x)
    vals, vecs = O.pca(cov)
    # the reference's fp64 fit differs from the oracle by rounding only; its fp32 fit by the fp32 rounding of its merge
    # and of eigh (eigenvalues to ~1e-7 of the largest, the top-16 eigenvectors to 1 - cos ~ 3e-7)
    for name, tol in (("fp64", 1e-10), ("fp32", 1e-5)):
        f = g["fits"][name]
        assert f["cov"].dtype == (torch.float64 if name == "fp64" else torch.float32)
        assert (f["mean"].double() - mean).abs().max() <= tol * mean.abs().max(), name
        assert (f["cov"].double() - cov).norm() <= tol * cov.norm(), name
        assert (f["eigvals"].double() - vals).abs().max() <= tol * vals.max(), name
        cos = (f["eigvecs"].double() * vecs).sum(dim=0).abs()[-16:]      # eigenvectors up to sign
        assert (cos >= 1 - tol).all(), (name, cos.min())
        assert torch.equal(f["trans"], f["mean"]) and torch.equal(f["rot"], f["eigvecs"])
        assert torch.allclose(f["scale"].double(), 1 / f["eigvals"].double().clamp(min=1e-6).sqrt(), rtol=1e-6)
    assert torch.allclose(O.get_dict(cov).abs(), g["fits"]["fp64"]["dict"].abs(), atol=1e-8)


def test_reference_pickles_load_here(golden):
    from sparse_coding_b200.learned_dict import Rotation, TiedSAE
    from sparse_coding_b200.pca import PCAEncoder
    from sparse_coding_b200.topk_encoder import TopKLearnedDict
    g = golden("pca")
    held = g["held"]
    kinds = {"pca_encoder": PCAEncoder, "rotation": Rotation, "topk": TopKLearnedDict, "pve_rotation": TiedSAE}
    for name, cls in kinds.items():
        e = g["exports"][name]
        ld = torch.load(io.BytesIO(e["pickle"]), weights_only=False)
        assert type(ld) is cls, name
        enc = ld.encode(ld.center(held))
        assert torch.allclose(enc, e["encode"], rtol=1e-5, atol=1e-6), name
        if "predict" in e:
            assert torch.allclose(ld.predict(held), e["predict"], rtol=1e-5, atol=1e-5), name
        assert pickle.dumps(ld).count(type(ld).__module__.encode()) >= 1
    assert PCAEncoder.__module__ == "autoencoders.pca" and Rotation.__module__ == "autoencoders.learned_dict"
    from autoencoders.learned_dict import Rotation as R2
    from autoencoders.pca import BatchedPCA, PCAEncoder as P2  # noqa: F401
    assert R2 is Rotation and P2 is PCAEncoder


def test_workspace_query_rejects_invalid_arguments():
    lib = _lib.load()
    ok = lib.sce_second_moments_workspace_bytes(512, 500)
    assert ok > 0
    assert lib.sce_second_moments_workspace_bytes(512, 65536) > ok
    for d, B in ((0, 10), (12, 10), (8200, 10), (512, 0), (512, -3), (512, (1 << 21) + 1)):
        assert lib.sce_second_moments_workspace_bytes(d, B) == 0, (d, B)


def test_workspace_need_never_decreases_with_rows():
    """A workspace sized for the longest call serves every shorter one, although the slice count of a call is not
    monotone in its rows (at d = 512, 64000 rows take 33 slices of 1984 rows and 65536 rows 32 of 2048)."""
    from sparse_coding_b200._rowpass import call_rows
    lib = _lib.load()
    for d in (8, 512, 2048):
        top = call_rows(d)
        needs = [lib.sce_second_moments_workspace_bytes(d, B) for B in range(1, top + 1)]
        assert all(n > 0 for n in needs)
        assert all(a <= b for a, b in zip(needs, needs[1:])), d
    assert lib.sce_second_moments_workspace_bytes(512, 64000) <= lib.sce_second_moments_workspace_bytes(512, 65536)


def test_abi_rejects_bad_arguments_without_device():
    lib = _lib.load()
    fake = C.c_void_p(1 << 20)                 # never dereferenced: every check runs before any CUDA call
    need = lib.sce_second_moments_workspace_bytes(64, 100)

    def call(x=fake, half=1, B=100, d=64, shift=fake, arith=0, col=fake, gram=fake, ws=fake, ws_bytes=need):
        return lib.sce_second_moments(x, half, B, d, shift, arith, col, gram, None, ws, ws_bytes, None)

    cases = [
        (dict(x=None), b"required"), (dict(shift=None), b"required"), (dict(col=None), b"required"),
        (dict(gram=None), b"required"), (dict(half=2), b"x_is_half"), (dict(B=0), b"outside"),
        (dict(d=60), b"multiple of 8"), (dict(d=8200), b"8192"), (dict(arith=5), b"unknown arith"),
        (dict(d=72, arith=_lib.SCE_ARITH_F16F8), b"multiple of 16"), (dict(x=C.c_void_p((1 << 20) + 8)), b"aligned"),
        (dict(ws_bytes=need - 1), b"workspace too small"), (dict(ws=C.c_void_p((1 << 20) + 512)), b"1024-byte"),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc in (-1, -3), (kw, rc)
        assert msg in lib.sce_last_error(), (kw, lib.sce_last_error())


def test_batched_pca_needs_a_cuda_device():
    from sparse_coding_b200.pca import BatchedPCA
    with pytest.raises(RuntimeError, match="CUDA device"):
        BatchedPCA(64, "cpu")
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA device"):
            BatchedPCA(64, "cuda:0")
