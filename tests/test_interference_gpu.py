"""The expected interference on the GPU: the drop-in against the reference's own calc_expected_interference (golden
fixture), and evaluate_dicts(interference=True) against the fp64 oracle applied to the code the engine holds, read back
with sce_read_code: the config-2 shape, ragged calls with guards past the outputs, mixed kinds with ICA's signed code,
top-k on both decode paths, rows with no active feature and rows whose active set spans several tiles, both
arithmetics, and every other key bitwise unchanged."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from interference_cases import cases, oracle_of_codes, rel_err
from oracle import baselines_oracle as BO
from oracle import top_fvu_oracle as TO
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def run_plan(key, lds, batches, arith="bf16x3"):
    """A _StatsPlan with the interference of every call, over ``batches`` (one call each): (cap_sums [M, n],
    nz_counts [M, n], [the code of every call, [M, B, n]])."""
    lib = _lib.load()
    with torch.cuda.device(DEV):
        p = MT._StatsPlan(key, lds, max(x.shape[0] for x in batches), arith, DEV, interference=True)
        try:
            codes = []
            for x in batches:
                p.run(x, 1, 0)
                code = torch.empty(p.M, x.shape[0], p.n, device=DEV)
                _lib.check(lib.sce_read_code(p.plan, x.shape[0], code.data_ptr(), p.stream), "sce_read_code")
                codes.append(code)
            torch.cuda.synchronize()
            return p.cap_sums.clone(), p.nz_counts.clone(), codes
        finally:
            p.close()


def check_against_oracle(ld, cap, nz, codes, m, tol=1e-5, margin=0.0):
    """Model m's sums against fp64 on its code; returns the fragile features (|totals| <= margin on some row)."""
    n = int(ld.n_feats)
    w = ld.get_learned_dict().to(DEV)
    want_cap, want_nz, fragile = oracle_of_codes(w, [c[m, :, :n] for c in codes], margin=margin)
    assert torch.equal(nz[m, :n], want_nz)
    keep = ~fragile
    assert rel_err(cap[m, :n][keep], want_cap[keep]) < tol
    assert (cap[m, n:] == 0).all() and (nz[m, n:] == 0).all()
    return fragile


def test_dropin_golden(golden):
    lib = _lib.load()
    for name, c in cases(golden).items():
        w, code = c["dictionary"].to(DEV), c["code"].to(DEV)
        got = S.calc_expected_interference(w, code)
        assert got.shape == c["expected"].shape and got.device == code.device and got.dtype == torch.float32
        assert rel_err(got, c["expected"]) < 1e-5, name
        assert torch.equal(got, S.calc_expected_interference(w, code)), name        # bitwise repeatable
        # the counts, exactly, from the plan-free entry point
        n, d = w.shape
        need = lib.sce_expected_interference_workspace_bytes(n, d, code.shape[0])
        ws, ptr = _lib.workspace(need, DEV, "sce_expected_interference_workspace_bytes")
        cap = torch.zeros(n + 4, dtype=torch.float64, device=DEV)
        nz = torch.full((n + 4,), -7, dtype=torch.int64, device=DEV)
        nz[:n] = 0
        cap[n:] = -7.0
        _lib.check(lib.sce_expected_interference(w.data_ptr(), n, d, code.data_ptr(), code.shape[0], cap.data_ptr(),
                                                 nz.data_ptr(), ptr, need, None), "sce_expected_interference")
        torch.cuda.synchronize()
        assert torch.equal(nz[:n].cpu(), c["nz_counts"]), name
        assert (nz[n:] == -7).all() and (cap[n:] == -7.0).all()


def test_dropin_dense_and_wide_rows():
    """Dense codes: hundreds of active features per row (several 64-feature tiles) at d = 512, rows with none, a d that
    is no multiple of 32, and more rows than one call takes. (Non-negative: a signed row with many active features
    almost always has some |totals| near 0, where no fp32 result is stable; ICA's signed code is checked below.)"""
    gen = torch.Generator().manual_seed(3)
    for n, d, B in ((600, 512, 300), (200, 50, 20000)):
        w = torch.randn(n, d, generator=gen)
        code = torch.rand(B, n, generator=gen) * (torch.rand(B, n, generator=gen) < 0.7)
        code[::7] = 0.0
        got = S.calc_expected_interference(w.to(DEV), code.to(DEV))
        cap, nz, _ = oracle_of_codes(w.to(DEV), [code.to(DEV)])
        assert rel_err(got, cap / nz.clamp(min=1)) < 1e-5, (n, d)


def _dicts(d, seed):
    """name -> LearnedDict: TiedSAE (sparse, and dense enough that a row's active set spans several 64-feature tiles),
    UntiedSAE, TopKLearnedDict on the dense decode (n = 48) and on the k-sparse gather (n = 1024 >= 96 k)."""
    gen = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen)
    unit = lambda w: w / w.norm(dim=-1, keepdim=True)
    return {"tied": S.TiedSAE(rn(96, d), rn(96) * 0.3 - 0.6),
            "tied_dense": S.TiedSAE(rn(512, d), rn(512) * 0.3 + 0.4),
            "untied": S.UntiedSAE(rn(96, d) * 0.5, rn(96, d), -(rn(96).abs() * 0.3 + 0.2)),
            "topk_dense": S.TopKLearnedDict(unit(rn(48, d)), 4),
            "topk_gather": S.TopKLearnedDict(unit(rn(1024, d)), 8)}


def _rows(N, d, seed):
    """[N, d] rows on the GPU, every 9th one zero (no active feature for the SAE kinds with negative biases)."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(N, d, generator=gen) * 0.8 + 0.1
    x[::9] = 0.0
    return x.to(DEV)


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_kinds_against_oracle_on_engine_code(arith):
    d = 64
    lds = _dicts(d, 5)
    batches = [_rows(B, d, B) for B in (1000, 37)]
    for name, ld in lds.items():
        n = int(ld.n_feats)
        kind = MT._eval_kind(ld)
        cap, nz, codes = run_plan((kind, n, d, False), [ld], batches, arith)
        check_against_oracle(ld, cap, nz, codes, 0)
        l0 = torch.cat([(c[0] != 0).sum(1) for c in codes])
        if name in ("tied", "untied"):
            assert (l0 == 0).any(), name                    # rows with no active feature (negative biases, x = 0)
        if name == "tied_dense":
            assert (l0 > 128).float().mean() > 0.5, l0.float().mean()   # rows spanning three tiles and more
        if kind == "topk":                                  # top-k: the activity mask holds the k selected features
            assert int(l0.max()) <= int(ld.sparsity)


@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_ica_signed_code(arith):
    bg = BO.load_golden()
    ica = BO.ica_from_golden(bg["ica"][0])
    d = int(ica.activation_size)
    x = _rows(3000, d, 2) * 2.0 + 0.5
    cap, nz, codes = run_plan(("ica", int(ica.n_feats), d, False), [ica], [x], arith)
    assert (codes[0] < 0).any()
    fragile = check_against_oracle(ica, cap, nz, codes, 0, margin=1e-3)
    assert fragile.float().mean() < 0.5


def test_mixed_kinds_and_other_keys_bitwise():
    """evaluate_dicts with ICA among SAE kinds: the interference of each against fp64 on its own code (a separate plan
    of the same rows), and every other key bitwise that of a call without interference."""
    bg = BO.load_golden()
    ica = BO.ica_from_golden(bg["ica"][0])
    d = int(ica.activation_size)
    lds = list(_dicts(d, 9).values())
    lds.insert(2, ica)
    x = _rows(9000, d, 4)
    plain = S.evaluate_dicts(lds, x)
    withi = S.evaluate_dicts(lds, x, interference=True)
    again = S.evaluate_dicts(lds, x, interference=True)
    for i, (a, b) in enumerate(zip(plain, withi)):
        assert set(b) == set(a) | {"expected_interference"}
        for k, v in a.items():
            assert (torch.equal(v, b[k]) or (torch.isnan(v).all() and torch.isnan(b[k]).all())) if torch.is_tensor(v) \
                else v == b[k], (i, k)
        ei = b["expected_interference"]
        assert ei.shape == (int(lds[i].n_feats),) and ei.dtype == torch.float32 and ei.device == x.device
        assert torch.equal(ei, again[i]["expected_interference"]), i
        ld = lds[i]
        kind = MT._eval_kind(ld)
        n = int(ld.n_feats)
        # the same row cuts as evaluate_dicts (segment 1000: calls of 8000 rows)
        _, _, codes = run_plan((kind, n, d, False), [ld], [x[:8000], x[8000:]])
        cap, nz, fragile = oracle_of_codes(ld.get_learned_dict().to(DEV), [c[0] for c in codes],
                                           margin=1e-3 if kind == "ica" else 0.0)
        want = cap / nz.clamp(min=1)
        assert torch.equal(b["feature_counts"].long(), nz) or kind == "ica", i
        assert rel_err(ei[~fragile], want[~fragile]) < 1e-5, (i, kind)


def test_config2_shape_against_fp64_oracle():
    """16 TiedSAE of 4096 features at d = 512 over 2^17 rows, about 50 active features per row."""
    M, n, d, N = 16, 4096, 512, 1 << 17
    gen = torch.Generator().manual_seed(2026)
    lds = [S.TiedSAE(torch.randn(n, d, generator=gen), torch.randn(n, generator=gen) * 0.1 - 2.25) for _ in range(M)]
    x = torch.randn(N, d, generator=torch.Generator().manual_seed(7)).to(DEV)
    r = S.evaluate_dicts(lds, x, interference=True)
    again = S.evaluate_dicts(lds, x, interference=True)
    rows = 8000
    batches = [x[s:s + rows] for s in range(0, N, rows)]
    cap, nz, codes = run_plan(("tied", n, d, False), lds, batches)
    l0 = float(sum((c[0] != 0).sum() for c in codes)) / N
    assert 20 < l0 < 120, l0
    for m in range(M):
        want_cap, want_nz, _ = oracle_of_codes(lds[m].get_learned_dict().to(DEV), [c[m] for c in codes])
        assert torch.equal(nz[m], want_nz), m
        assert rel_err(cap[m], want_cap) < 1e-5, m
        want = want_cap / want_nz.clamp(min=1)
        assert rel_err(r[m]["expected_interference"], want) < 1e-5, m
        assert torch.equal(r[m]["expected_interference"], again[m]["expected_interference"]), m
    del codes


def test_ragged_calls_and_guards():
    """One sce_code_interference call per row count, accumulating, with guard values past both outputs."""
    d = 64
    lds = [S.TiedSAE(torch.randn(96, d), torch.randn(96) * 0.3 - 0.4) for _ in range(3)]
    lib = _lib.load()
    with torch.cuda.device(DEV):
        p = MT._StatsPlan(("tied", 96, d, False), lds, 200, "bf16x3", DEV)
        try:
            need = lib.sce_interference_workspace_bytes(C.byref(p.desc), 200)
            ws = torch.full((need // 4 + 256,), float("nan"), device=DEV)
            base = C.c_void_p(ws.data_ptr() + (-ws.data_ptr()) % 1024)
            cap = torch.full((3 * 96 + 5,), -7.0, dtype=torch.float64, device=DEV)
            nz = torch.full((3 * 96 + 5,), -7, dtype=torch.int64, device=DEV)
            cap[:288], nz[:288] = 0.0, 0
            codes = []
            for B in (1, 33, 200, 7):
                x = torch.randn(B, d, device=DEV)
                p.run(x, 1, 0)
                rc = lib.sce_code_interference(p.plan, B, cap.data_ptr(), nz.data_ptr(), base, need, p.stream)
                assert rc == 0, lib.sce_last_error().decode()
                code = torch.empty(3, B, 96, device=DEV)
                _lib.check(lib.sce_read_code(p.plan, B, code.data_ptr(), p.stream), "sce_read_code")
                codes.append(code)
            torch.cuda.synchronize()
            assert (cap[288:] == -7.0).all() and (nz[288:] == -7).all()
            check_against_oracle(lds[0], cap[:288].view(3, 96), nz[:288].view(3, 96), codes, 0)
            for m in (1, 2):
                check_against_oracle(lds[m], cap[:288].view(3, 96), nz[:288].view(3, 96), codes, m)
        finally:
            p.close()


def test_abi_refusals():
    lib = _lib.load()
    d = 32
    lds = [S.TiedSAE(torch.randn(32, d), torch.zeros(32))] * 2
    with torch.cuda.device(DEV):
        p = MT._StatsPlan(("tied", 32, d, False), lds, 64, "bf16x3", DEV)
        try:
            x = torch.randn(64, d, device=DEV)
            p.run(x, 1, 0)
            need = lib.sce_interference_workspace_bytes(C.byref(p.desc), 64)
            ws, ptr = _lib.workspace(need, DEV, "sce_interference_workspace_bytes")
            cap = torch.zeros(2, 32, dtype=torch.float64, device=DEV)
            nz = torch.zeros(2, 32, dtype=torch.int64, device=DEV)
            call = lambda B=64, c=cap.data_ptr(), z=nz.data_ptr(), w=ptr, nb=need: \
                (lib.sce_code_interference(p.plan, B, c, z, w, nb, p.stream), lib.sce_last_error().decode())
            assert call()[0] == 0
            torch.cuda.synchronize()
            before = (cap.clone(), nz.clone())
            for kw, rc, msg in ((dict(B=0), -1, "B = 0"), (dict(B=65), -1, "B = 65"), (dict(c=None), -1, "required"),
                                (dict(z=None), -1, "required"), (dict(nb=need - 1), -3, "workspace too small"),
                                (dict(w=ptr + 512), -3, "aligned")):
                got, err = call(**kw)
                assert got == rc and msg in err, (kw, got, err)
            torch.cuda.synchronize()
            assert torch.equal(cap, before[0]) and torch.equal(nz, before[1])
        finally:
            p.close()
