"""The top- and rest-feature FVU on the GPU (evaluate_dicts(n_top=...), fraction_variance_unexplained_top_activating,
sce_forward_split): parity with the reference's own function on the golden fixture, the other keys bitwise those of a
call without n_top, mixed kinds in one call, fp16 and CPU-resident activations, both arithmetics, top-k on the gather and
the dense-decode path, a centred TiedSAE, the config-2 shape against the fp64 oracle, repeatability, and the ABI's
refusals."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from oracle import baselines_oracle as BO
from oracle import top_fvu_oracle as TO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.learned_dict import IdentityReLU, RandomDict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def engine_dict(e):
    k = e["kind"]
    if k == "tied":
        return S.TiedSAE(e["encoder"], e["encoder_bias"],
                         centering=(e.get("center_trans"), e.get("center_rot"), e.get("center_scale")))
    if k == "untied":
        return S.UntiedSAE(e["encoder"], e["decoder"], e["encoder_bias"])
    if k == "topk":
        return S.TopKLearnedDict(e["dict"], e["sparsity"])
    n, d = e["encoder"].shape
    if k == "random":
        rd = RandomDict(d, n)
        rd.encoder, rd.encoder_bias = e["encoder"].clone(), e["encoder_bias"].clone()
        return rd
    ir = IdentityReLU(d)
    ir.bias = e["encoder_bias"].clone()
    return ir


def oracle_dict(e):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in e.items()}


def width(e):
    return (e["dict"] if e["kind"] == "topk" else e["encoder"]).shape[1]


def rel(a, b):
    return abs(float(a) / float(b) - 1.0)


@pytest.mark.parametrize("arith,tol", [("bf16x3", 1e-4), ("f16f8", 2e-3)])
def test_golden_parity(golden, arith, tol):
    g = golden("top_fvu")
    for c in g["cases"]:
        e = g["dicts"][c["dict"]]
        x = TO.rows(width(e), c["x_seed"]).to(DEV)
        top, rest = S.fraction_variance_unexplained_top_activating(engine_dict(e), x, n_top=c["n_top"], arith=arith)
        assert top.dim() == 0 and top.device == x.device
        assert rel(top, c["fvu_top"]) < tol and rel(rest, c["fvu_rest"]) < tol, (c["dict"], c["n_top"], float(top),
                                                                                 c["fvu_top"], float(rest), c["fvu_rest"])
        r = S.evaluate_dicts([engine_dict(e)], x, n_top=c["n_top"], arith=arith)[0]
        assert torch.equal(r["top_features"].cpu(), c["top_features"]), c["dict"]
        assert r["fvu_top"] == top and r["fvu_rest"] == rest


@pytest.mark.parametrize("where,dtype", [("cuda", torch.float32), ("cpu", torch.float16)])
def test_mixed_kinds_and_other_keys_bitwise(golden, where, dtype):
    g = golden("top_fvu")
    names = ["tied_identity", "tied_centred", "topk", "identity_relu"]
    lds = [engine_dict(g["dicts"][k]) for k in names]
    bg = BO.load_golden()
    ica = BO.ica_from_golden(bg["ica"][0])
    lds.insert(2, ica)
    x = TO.rows(32, 1).to(dtype)
    x = x.pin_memory() if where == "cpu" else x.to(DEV)
    plain = S.evaluate_dicts(lds, x)
    split = S.evaluate_dicts(lds, x, n_top=2)
    xd = x.double().to(DEV)
    for i, (a, b) in enumerate(zip(plain, split)):
        assert set(b) == set(a) | {"top_features", "fvu_top", "fvu_rest"}
        for k, v in a.items():
            assert (torch.equal(v, b[k]) or (torch.isnan(v).all() and torch.isnan(b[k]).all())) if torch.is_tensor(v) \
                else v == b[k], (i, k)
        assert b["fvu_top"].device == x.device and b["top_features"].dtype == torch.int64
    assert torch.isnan(split[2]["fvu_top"]) and torch.isnan(split[2]["fvu_rest"])
    assert split[2]["top_features"].unique().numel() == 2
    for i, name in zip((0, 1, 3, 4), names):
        m = BO.to(oracle_dict(g["dicts"][name]), DEV)
        top, rest, feats = TO.fraction_variance_unexplained_top_activating(m, xd, 2)
        assert torch.equal(split[i]["top_features"].to(DEV), feats), name
        assert rel(split[i]["fvu_top"], top) < 1e-4 and rel(split[i]["fvu_rest"], rest) < 1e-4, name


def test_centred_tied_uses_center_not_uncenter(golden):
    g = golden("top_fvu")
    e = g["dicts"]["tied_centred"]
    assert engine_dict(e) is not None and MT._is_centred(engine_dict(e))
    c = [c for c in g["cases"] if c["dict"] == "tied_centred" and c["n_top"] == 5][0]
    x = TO.rows(32, c["x_seed"]).to(DEV)
    top, rest = S.fraction_variance_unexplained_top_activating(engine_dict(e), x, n_top=5)
    assert rel(top, c["fvu_top"]) < 1e-4 and rel(rest, c["fvu_rest"]) < 1e-4


def _planted_tied(M, n, d, n_top, seed):
    """M TiedSAE with n_top features per model raised by a bias of +0.5: a wide gap at rank n_top."""
    gen = torch.Generator().manual_seed(seed)
    lds, ms = [], []
    for _ in range(M):
        enc = torch.randn(n, d, generator=gen)
        b = torch.randn(n, generator=gen) * 0.1 - 0.3
        b[torch.randperm(n, generator=gen)[:n_top]] += 0.5
        lds.append(S.TiedSAE(enc, b))
        ms.append({"kind": "tied", "encoder": enc.double().to(DEV), "encoder_bias": b.double().to(DEV)})
    return lds, ms


def _oracle_chunked(m, x, n_top, rows=16384):
    """fp64 (fvu_top, fvu_rest, top) of oracle dictionary ``m`` on [N, d] ``x`` in row chunks."""
    w = TO.decoder(m)
    s = sum(TO.code(m, x[i:i + rows].double()).sum(0) for i in range(0, x.shape[0], rows))
    top = torch.sort(s, descending=True, stable=True).indices[:n_top]
    keep = torch.zeros(s.shape[0], dtype=torch.bool, device=x.device)
    keep[top] = True
    st = sr = 0.0
    for i in range(0, x.shape[0], rows):
        xc = x[i:i + rows].double()
        c = TO.code(m, xc)
        st += float((xc - (c * keep) @ w).pow(2).sum())
        sr += float((xc - (c * ~keep) @ w).pow(2).sum())
    xd = x.double()
    tot = float((xd - xd.mean(0)).pow(2).sum())
    return st / tot, sr / tot, top


def test_topk_gather_and_dense_paths():
    torch.manual_seed(5)
    d, N = 64, 20000
    x = (torch.randn(N, d) * 0.8 + 0.2).to(DEV)
    for n in (48, 1024):            # 1024 >= 96 * 8: the k-sparse gather kernel decodes; 48: the dense GEMM
        gen = torch.Generator().manual_seed(n)
        w = torch.randn(n, d, generator=gen)
        w = w / w.norm(dim=-1, keepdim=True)      # (TopKLearnedDict is stored normalised)
        ld = S.TopKLearnedDict(w, 4)
        m = {"kind": "topk", "dict": w.double().to(DEV), "sparsity": 4}
        c = TO.code(m, x.double())
        top_mean = float(c.mean(0).abs().max())
        gap = TO.mean_gap(c, 3) / top_mean
        assert gap > 1e-4, gap
        r = S.evaluate_dicts([ld], x, n_top=3)[0]
        top, rest, feats = TO.fraction_variance_unexplained_top_activating(m, x.double(), 3)
        assert torch.equal(r["top_features"], feats), n
        assert rel(r["fvu_top"], top) < 1e-4 and rel(r["fvu_rest"], rest) < 1e-4, (n, float(r["fvu_top"]), float(top))


def test_config2_shape_against_fp64_oracle():
    M, n, d, N, k = 16, 4096, 512, 1 << 17, 2
    lds, ms = _planted_tied(M, n, d, k, 2026)
    gen = torch.Generator().manual_seed(7)
    x = (torch.randn(N, d, generator=gen) * 0.7).to(DEV)
    r = S.evaluate_dicts(lds, x, n_top=k)
    again = S.evaluate_dicts(lds, x, n_top=k)
    for i in range(M):
        top, rest, feats = _oracle_chunked(ms[i], x, k)
        assert torch.equal(r[i]["top_features"], feats), i
        assert rel(r[i]["fvu_top"], top) < 1e-4 and rel(r[i]["fvu_rest"], rest) < 1e-4, (i, float(r[i]["fvu_top"]), top,
                                                                                        float(r[i]["fvu_rest"]), rest)
        assert torch.equal(r[i]["fvu_top"], again[i]["fvu_top"]) and torch.equal(r[i]["fvu_rest"], again[i]["fvu_rest"])


def test_ragged_calls_and_guards():
    """Ragged B, NaN rows past B and guard values past every output: one sce_forward_split call per row count."""
    lds, ms = _planted_tied(3, 96, 64, 2, 11)
    key = ("tied", 96, 64, False)
    lib = _lib.load()
    with torch.cuda.device(DEV):
        p = MT._StatsPlan(key, lds, 200, "bf16x3", DEV)
        try:
            p.start_split(torch.tensor([[0, 1], [5, 2], [95, 40]], device=DEV))
            for B in (1, 33, 200):
                xs = torch.full((200, 64), float("nan"), device=DEV)
                xs[:B] = torch.randn(B, 64, device=DEV)
                out = torch.full((2, 5), -7.0, dtype=torch.float64, device=DEV)
                out[0, :3] = 0.0
                out[1, :3] = 0.0
                ws = torch.full((p.split_bytes // 4 + 256,), float("nan"), device=DEV)
                base = ws.data_ptr() + (-ws.data_ptr()) % 1024
                rc = lib.sce_forward_split(p.plan, xs.data_ptr(), B, 2, p.top_cols.data_ptr(), out[0].data_ptr(),
                                           out[1].data_ptr(), None, None, C.c_void_p(base), p.split_bytes, p.stream)
                assert rc == 0, lib.sce_last_error().decode()
                assert (out[:, 3:] == -7.0).all()
                for m in range(3):
                    mm = ms[m]
                    xd = xs[:B].double()
                    c = TO.code(mm, xd)
                    keep = torch.zeros(96, dtype=torch.bool, device=DEV)
                    keep[p.top_cols[m].long()] = True
                    w = TO.decoder(mm)
                    want_t = float((xd - (c * keep) @ w).pow(2).sum())
                    want_r = float((xd - (c * ~keep) @ w).pow(2).sum())
                    assert abs(float(out[0, m]) - want_t) <= 1e-4 * want_t + 1e-6, (B, m)
                    assert abs(float(out[1, m]) - want_r) <= 1e-4 * want_r + 1e-6, (B, m)
        finally:
            p.close()


def test_abi_refusals(golden):
    lib = _lib.load()
    lds, _ = _planted_tied(2, 32, 32, 2, 3)
    g = golden("top_fvu")
    cen = [engine_dict(g["dicts"]["tied_centred"])] * 2
    with torch.cuda.device(DEV):
        plain = MT._StatsPlan(("tied", 32, 32, False), lds, 64, "bf16x3", DEV)
        centred = MT._StatsPlan(("tied", 48, 32, True), cen, 64, "bf16x3", DEV)
        try:
            x = torch.randn(64, 32, device=DEV)
            sq = torch.zeros(2, 2, dtype=torch.float64, device=DEV)
            xh = torch.zeros(2, 64, 32, device=DEV)

            def call(p, cols, n_top=2, x_hat=None, x_hat_top=None):
                need = lib.sce_forward_split_workspace_bytes(C.byref(p.desc), 64, 2)
                ws, ptr = _lib.workspace(need, DEV, "sce_forward_split_workspace_bytes")
                c = torch.tensor(cols, dtype=torch.int32, device=DEV)
                rc = lib.sce_forward_split(p.plan, x.data_ptr(), 64, n_top, c.data_ptr(), sq[0].data_ptr(),
                                           sq[1].data_ptr(), x_hat, x_hat_top, ptr, need, p.stream)
                return rc, lib.sce_last_error().decode() if rc else ""

            assert call(plain, [[0, 1], [2, 3]])[0] == 0
            before = sq.clone()
            for cols, n_top, msg in (([[0, 1], [2, 3]], 0, "n_top = 0"), ([[0, 1], [2, 3]], 65, "n_top = 65"),
                                     ([[0, 32], [2, 3]], 2, "outside [0, n = 32)"), ([[0, 1], [-1, 3]], 2, "outside"),
                                     ([[0, 1], [3, 3]], 2, "column 3 appears twice in top_cols[1]")):
                rc, err = call(plain, cols, n_top)
                assert rc == -1 and msg in err, (cols, n_top, err)
            assert torch.equal(sq, before)
            rc, err = call(centred, [[0, 1], [2, 3]], x_hat=xh.data_ptr())
            assert rc == -1 and "needs x_hat and x_hat_top" in err
            assert call(centred, [[0, 1], [2, 3]], x_hat=xh.data_ptr(), x_hat_top=torch.zeros_like(xh).data_ptr())[0] == 0
            assert torch.equal(sq, before)
        finally:
            plain.close()
            centred.close()
