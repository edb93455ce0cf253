"""ICAEncoder on the GPU: one sce_ica_pass against fp64 on the device at widths 32 to 2048, both arithmetics and input
types; the pass's properties (call splitting, bitwise repeatability, tanh saturation, padding rows, the f16f8 range
flag); full fits against oracle/ica_oracle.py from the same w_init and against the reference's fits in
tests/golden/ica.pt; recovery of known sources; the properties the reference's test/test_ica.py checks; the exports.
Each test prints the deviations it observed; the bars hold at least 3x over what an H100 showed."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

import sparse_coding_b200 as S
from oracle import eval_oracle as EO
from oracle import ica_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ica import ICAEncoder

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ARITHS = ["bf16x3", "f16f8"]


def ica_pass(x, shift, unmix, alpha=1.0, arith="bf16x3", flag=None, g_sum=None, gx=None, rows=None):
    """g_sum, gx (fp64, accumulated into the given ones) of sce_ica_pass over ``x`` in calls of ``rows`` rows."""
    lib = _lib.load()
    B, d = x.shape
    n = unmix.shape[0]
    g_sum = torch.zeros(n, dtype=torch.float64, device=DEV) if g_sum is None else g_sum
    gx = torch.zeros(n, d, dtype=torch.float64, device=DEV) if gx is None else gx
    rows = rows or B
    ws, ptr = _lib.workspace(lib.sce_ica_pass_workspace_bytes(d, n, min(rows, B)), DEV, "sce_ica_pass_workspace_bytes")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for s in range(0, B, rows):
        xb = x[s:s + rows].contiguous()
        _lib.check(lib.sce_ica_pass(xb.data_ptr(), int(x.dtype == torch.float16), xb.shape[0], d, shift.data_ptr(),
                                    unmix.data_ptr(), n, C.c_float(alpha), _lib.arith_code(arith), g_sum.data_ptr(),
                                    gx.data_ptr(), flag.data_ptr() if flag is not None else None, ptr,
                                    ws.numel() - 1024, stream), "sce_ica_pass")
    torch.cuda.synchronize()
    return g_sum, gx


def pass64(x, shift, unmix, alpha=1.0):
    v = x.double() - shift.double()
    t = torch.tanh(alpha * (v @ unmix.double().T))
    return (alpha * (1 - t * t)).sum(dim=0), t.T @ v


def operands(B, d, n, dtype, seed, offset=3.0, gain=2.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    mu = offset * torch.randn(d, generator=g, device=DEV)
    x = (torch.randn(B, d, generator=g, device=DEV) + mu).to(dtype)
    shift = (mu + 0.1 * torch.randn(d, generator=g, device=DEV)).contiguous()   # independent of x: B = 1 has v != 0
    unmix = (gain / d ** 0.5) * torch.randn(n, d, generator=g, device=DEV)
    return x, shift, unmix


def rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("d,n", [(32, 32), (128, 128), (512, 512), (2048, 2048), (512, 256)])
def test_pass_against_fp64(d, n, arith, dtype):
    worst = [0.0, 0.0]
    for i, B in enumerate((1, 63, 2049, 65536)):
        x, shift, unmix = operands(B, d, n, dtype, seed=100 * d + i)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        g_sum, gx = ica_pass(x, shift, unmix, 1.0, arith, flag)
        g64, gx64 = pass64(x, shift, unmix)
        assert int(flag.item()) == 0
        e_gx, e_g = rel(gx, gx64), rel(g_sum, g64)
        worst = [max(worst[0], e_gx), max(worst[1], e_g)]
        print(f"d={d} n={n} {arith} {dtype} B={B}: gx {e_gx:.2e}  g_sum {e_g:.2e}")
        assert e_gx <= 1.5e-4 and e_g <= 1.5e-4, (B, e_gx, e_g)
    print(f"worst: gx {worst[0]:.2e}  g_sum {worst[1]:.2e}")


@pytest.mark.parametrize("arith", ARITHS)
def test_pass_properties(arith):
    d, n = 512, 512
    x, shift, unmix = operands(4096, d, n, torch.float32, seed=7)
    whole = ica_pass(x, shift, unmix, 1.5, arith)
    again = ica_pass(x, shift, unmix, 1.5, arith)
    assert torch.equal(whole[0], again[0]) and torch.equal(whole[1], again[1]), "not bitwise repeatable"
    # 2048-row calls cut the rows into the same 256-row slices: only the fp64 order of the partial sums differs
    parts = ica_pass(x, shift, unmix, 1.5, arith, rows=2048)
    e = max(rel(parts[0], whole[0]), rel(parts[1], whole[1]))
    print(f"{arith}: split calls {e:.2e}")
    assert e <= 1e-13
    # saturation: at |u| ~ 1e3 t is sign(u) and g' vanishes but for the few u near 0
    big = unmix * 1e3
    g_sum, gx = ica_pass(x, shift, big, 1.0, arith)
    g64, gx64 = pass64(x, shift, big)
    e_sat = rel(gx, gx64)
    print(f"{arith}: saturated gx {e_sat:.2e}  g_sum / B {float(g_sum.max()) / 4096:.2e} (fp64 {float(g64.max()) / 4096:.2e})")
    assert e_sat <= (2e-4 if arith == "bf16x3" else 1e-3) and float(g_sum.max()) <= 1e-2 * 4096
    assert float((g_sum - g64).abs().max()) <= 1e-3 * 4096
    # padding rows add nothing: with unmix = 0 every real row adds alpha to each g_sum entry, and nothing else does
    for B in (1, 63, 100):
        g_sum, gx = ica_pass(x[:B], shift, torch.zeros_like(unmix), 1.25, arith)
        assert torch.equal(g_sum, torch.full_like(g_sum, 1.25 * B)), (B, g_sum[:4])
        assert float(gx.abs().max()) == 0.0


def test_f16f8_range_flag_covers_rows_and_unmix():
    d = n = 64
    x, shift, unmix = operands(300, d, n, torch.float32, seed=8)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    ica_pass(x, shift, unmix, 1.0, "f16f8", flag)
    assert int(flag.item()) == 0
    xb = x.clone()
    xb[17, 5] = 1e5
    ica_pass(xb, shift, unmix, 1.0, "f16f8", flag)
    assert int(flag.item()) == 1
    flag.zero_()
    ub = unmix.clone()
    ub[3, 9] = 7e4
    ica_pass(x, shift, ub, 1.0, "f16f8", flag)
    assert int(flag.item()) == 1
    flag.zero_()
    ica_pass(xb, shift, unmix, 1.0, "bf16x3", flag)   # no range check outside f16f8
    assert int(flag.item()) == 0


def w_init_for(d, seed):
    return np.random.RandomState(seed).normal(size=(d, d))


def oracle_fit(x, w_init, **kw):
    return O.fit(x.to(DEV).float().double(), torch.from_numpy(w_init).to(DEV), **kw)


def comp_err(ica, r):
    c = torch.from_numpy(ica.ica.components_).to(DEV)
    return rel(c, r["components"])


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("d,N", [(64, 16000), (512, 65536)])
def test_early_iterations_against_oracle(d, N, arith):
    x, _ = O.mixed_sources(d, N, seed=d)
    w = w_init_for(d, 1)
    # at d = 512 the update matrix's singular values spread over four decades within three iterations (from random
    # starts FastICA's early updates are ill-conditioned), so its small directions amplify any rounding: compared there
    # after one iteration only
    for it in (1, 3) if d == 64 else (1,):
        ica = ICAEncoder(d, device=DEV, arith=arith, max_iter=it, w_init=w)
        with pytest.warns(UserWarning, match="did not converge"):
            ica.fit(x.to(DEV))
        r = oracle_fit(x, w, max_iter=it)
        e = comp_err(ica, r)
        print(f"d={d} {arith} after {it} iterations: components {e:.2e}")
        # from a random start the projections are near-Gaussian, and the update's two terms, E[g(u) x] and E[g'(u)] w,
        # nearly cancel: the pass's ~1e-5 becomes ~1e-3 in the first iterates (the converged fits land ~1e-5 from fp64)
        assert ica.ica.n_iter_ == it and e <= 1e-2


@pytest.mark.parametrize("name", ["mixed32", "mixed64"])
def test_fixture_fits(golden, name):
    g = golden("ica")
    f = g["fits"][name]
    rows, _ = O.mixed_sources(f["d"], f["n"] + g["held_rows"], f["data_seed"])
    x, held = rows[:f["n"]], rows[f["n"]:]
    ica = ICAEncoder(f["d"], device=DEV, w_init=f["w_init"].numpy())
    src = ica.train(x)           # fp64 rows: fitted as fp32
    t = lambda a: torch.from_numpy(np.asarray(a))
    errs = {"components": rel(t(ica.ica.components_), f["ica"]["components"]),
            "mixing": rel(t(ica.ica.mixing_), f["ica"]["mixing"]),
            "whitening": rel(t(ica.ica.whitening_), f["ica"]["whitening"]),
            "scaler_mean": rel(t(ica.scaler.mean_), f["scaler"]["mean"]),
            "scaler_scale": rel(t(ica.scaler.scale_), f["scaler"]["scale"]),
            "train_sources": rel(src[:g["held_rows"]], f["train_sources_head"]),
            "held_sources": rel(ica.encode(held), f["held_sources"])}
    print(name, "n_iter", ica.ica.n_iter_, f["n_iter"], {k: f"{v:.2e}" for k, v in errs.items()})
    assert src.dtype == torch.float64 and src.device == x.device
    assert all(v <= 1e-4 for v in errs.values()), errs
    if f["lims"][-1] <= 1e-5 and all(l >= 3e-4 for l in f["lims"][:-1]):
        assert ica.ica.n_iter_ == f["n_iter"]


def test_large_offset_with_an_outlier_first_row():
    d, N = 64, 20000
    x, _ = O.mixed_sources(d, N, seed=17)
    x = x + 1e3
    c = x.mean(dim=0)
    x[0] = c + 10.0 * (x[0] - c)                             # a BOS-like outlier: 10x the row's deviation
    w = w_init_for(d, 2)
    ica = ICAEncoder(d, device=DEV, w_init=w)
    ica.fit(x.float().to(DEV))
    r = oracle_fit(x, w)
    e = comp_err(ica, r)
    print(f"offset 1e3 + outlier row: n_iter {ica.ica.n_iter_} / {r['n_iter']}, components {e:.2e}")
    assert e <= 1e-3


def laplace(N, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = (torch.rand(N, d, generator=g, device=DEV) - 0.5).clamp_(min=-0.4999999)   # rand() can be 0: log1p(-1) = -inf
    return -torch.sign(u) * torch.log1p(-2 * u.abs()), g


def test_recovers_known_sources():
    d, N = 512, 1 << 20
    s, g = laplace(N, d, seed=5)
    A = 0.3 * torch.randn(d, d, generator=g, device=DEV, dtype=torch.float64) / d ** 0.5 + torch.eye(
        d, device=DEV, dtype=torch.float64)   # singular values within about [0.4, 1.6]
    x = (s.double() @ A.T + 3.0).float()
    del s
    np.random.seed(0)
    ica = ICAEncoder(d, device=DEV)
    ica.fit(x)
    est = torch.from_numpy(ica.ica.components_).to(DEV) / torch.from_numpy(ica.scaler.scale_).to(DEV)
    true = torch.linalg.inv(A)
    cos = (true / true.norm(dim=1, keepdim=True)) @ (est / est.norm(dim=1, keepdim=True)).T
    best = cos.abs().max(dim=1).values
    print(f"d={d} N={N}: n_iter {ica.ica.n_iter_}, worst |cos| {float(best.min()):.5f}, median {float(best.median()):.5f}")
    assert float(best.min()) >= 0.99


def test_reference_test_ica_properties():
    """test/test_ica.py restated at d = 8 (the engine's smallest width)."""
    rs = np.random.RandomState(0)
    X = torch.tensor(rs.laplace(0, 1, (4000, 8)))
    ica = ICAEncoder(8, device=DEV)
    out = ica.train(X)
    assert torch.allclose(out, ica.encode(X), atol=1e-5)
    comps = ica.ica.components_ / np.linalg.norm(ica.ica.components_, axis=1)[:, None]
    comps = comps[np.argsort(np.abs(comps).argmax(axis=1))]
    print("identity recovery: max | |comps| - I |", float(np.abs(np.abs(comps) - np.eye(8)).max()))
    assert np.allclose(np.abs(comps), np.eye(8), atol=1e-1)
    # non-Gaussian: two fits from different starts agree up to permutation and sign; Gaussian: they do not
    def two_fits(X):
        a, b = ICAEncoder(X.shape[1], device=DEV), ICAEncoder(X.shape[1], device=DEV)
        np.random.seed(1)
        oa = a.train(X)
        np.random.seed(2)
        ob = b.train(X)
        return a, b, oa, ob
    X = torch.tensor(np.random.RandomState(42).laplace(0, 1, (4000, 8)))
    a, b, oa, ob = two_fits(X)
    ca, cb = np.abs(a.ica.components_), np.abs(b.ica.components_)
    pa, pb = ca.argmax(axis=1).argsort(), cb.argmax(axis=1).argsort()
    print("non-Gaussian: max component difference", float(np.abs(ca[pa] - cb[pb]).max()))
    assert np.allclose(ca[pa], cb[pb], atol=5e-3)   # both stop within tol = 1e-4 of the same fixed point
    assert torch.allclose(oa[:, pa].abs(), ob[:, pb].abs(), atol=1e-2)
    X = torch.tensor(np.random.RandomState(42).randn(4000, 8))
    _, _, oa, ob = two_fits(X)
    assert not torch.allclose(oa, ob, atol=1e-5)


def test_exports():
    d = 64
    x, _ = O.mixed_sources(d, 20000, seed=31)
    xd = x.float().to(DEV)
    np.random.seed(3)
    ica = ICAEncoder(d, device=DEV)
    src = ica.train(xd)
    assert src.device == xd.device and torch.equal(src, ica.encode(xd))
    held = O.mixed_sources(d, 4000, seed=31)[0][-4000:].float().to(DEV)
    lds = [ica.to_topk_dict(k) for k in (1, 4, 16)]
    for ld in lds:
        ld.to_device(DEV)
    res = MT.evaluate_dicts(lds, held)
    hd = held.double()
    for ld, r in zip(lds, res):
        m = {"kind": "topk", "dict": ld.dict.double(), "sparsity": int(ld.sparsity)}
        fvu = float(EO.fraction_variance_unexplained(m, hd))
        pred = ld.predict(held).double()
        own = float(((pred - hd) ** 2).sum() / ((hd - hd.mean(dim=0)) ** 2).sum())
        print(f"topk {ld.sparsity}: engine fvu {float(r['fvu']):.6f}  oracle {fvu:.6f}  own predict {own:.6f}")
        assert abs(float(r["fvu"]) - fvu) <= 1e-4 * fvu
        assert abs(own - fvu) <= 1e-4 * fvu


def test_reference_pickle_encodes_on_the_device(golden):
    pytest.importorskip("sklearn")
    g = golden("ica")
    f = g["fits"]["mixed32"]
    held = O.mixed_sources(32, f["n"] + g["held_rows"], f["data_seed"])[0][f["n"]:]
    ica = torch.load(io.BytesIO(f["pickle"]), weights_only=False)
    out = ica.encode(held.to(DEV))
    assert out.device.type == "cuda" and torch.allclose(out.cpu(), f["held_sources"], rtol=1e-12, atol=1e-12)


def test_rank_deficient_input_raises():
    x, _ = O.mixed_sources(32, 5000, seed=4)
    x[:, 7] = x[:, 3]
    with pytest.raises(ValueError, match="rank-deficient"):
        ICAEncoder(32, device=DEV).fit(x.to(DEV))
    x[:, 7] = 5.0
    with pytest.raises(ValueError, match="rank-deficient"):
        ICAEncoder(32, device=DEV).fit(x.to(DEV))
    x[5, 2] = float("inf")
    with pytest.raises(ValueError, match="non-finite"):
        ICAEncoder(32, device=DEV).fit(x.to(DEV))
