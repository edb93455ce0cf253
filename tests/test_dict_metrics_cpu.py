"""Dictionary-similarity metrics without a GPU: the golden fixture (the reference's own standard_metrics results)
against the fp64 restatement in oracle/metrics_oracle.py, argument validation of the sce_similarity ABI, its workspace
bound at config 5, and the learned-dictionary description of every signature."""
import ctypes as C

import pytest
import torch

import sparse_coding_b200 as S
from oracle import metrics_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ensemble import stack_dict


def oracle_arg(golden_dicts, name):
    if isinstance(name, list):
        return [oracle_arg(golden_dicts, x) for x in name]
    e = golden_dicts[name]
    return O.learned(e["kind"], e["w"])


def test_golden_matches_fp64_oracle(golden):
    g = golden("dict_metrics")
    assert len(g["cases"]) >= 50
    for c in g["cases"]:
        args = [oracle_arg(g["dicts"], a) for a in c["args"]]
        want = O.FUNCS[c["fn"]](*args)
        got = c["out"].double()
        assert got.shape == want.shape, c["fn"]
        assert torch.equal(torch.isnan(got), torch.isnan(want)), (c["fn"], c["args"])
        ok = ~torch.isnan(want)
        assert torch.allclose(got[ok], want[ok], rtol=1e-5, atol=2e-6), (c["fn"], c["args"], (got - want)[ok].abs().max())


def test_golden_covers_the_edge_cases(golden):
    g = golden("dict_metrics")
    kinds = {e["kind"] for e in g["dicts"].values()}
    assert {"tied", "untied", "topk", "raw"} <= kinds
    shapes = [tuple(e["w"].shape) for e in g["dicts"].values()]
    assert any(n == 8 and d == 8 for n, d in shapes) and any(n % 128 and d % 16 for n, d in shapes)
    neg = [c for c in g["cases"] if c["fn"] == "mcs_duplicates" and c["args"] == ["pos", "neg"]][0]
    assert (neg["out"] < 0).all()                                   # every cosine negative: a zero row must not win
    cap = [c for c in g["cases"] if c["fn"] == "capacity_per_feature" and c["args"] == ["zero_row"]][0]
    assert torch.isnan(cap["out"][5]) and not torch.isnan(cap["out"][:5]).any()


def _call(lib, **kw):
    a = dict(a=1 << 20, ma=2, na=64, a_rows=None, a_floor=1e-8, a_norm=1, b=None, mb=0, nb=0, b_rows=None, b_floor=0.0,
             b_norm=1, d=64, pairs=[(1, 0)], arith=_lib.SCE_ARITH_AUTO, row=1 << 21, col=1 << 22, cap=None,
             ws=1 << 30, ws_bytes=1 << 40)
    a.update(kw)
    ints = lambda v: (C.c_int * len(v))(*v) if v is not None else None
    pv = [x for p in a["pairs"] for x in p] if a["pairs"] is not None else None
    rc = lib.sce_similarity(a["a"], a["ma"], a["na"], ints(a["a_rows"]), C.c_float(a["a_floor"]), a["a_norm"], a["b"],
                            a["mb"], a["nb"], ints(a["b_rows"]), C.c_float(a["b_floor"]), a["b_norm"], a["d"], ints(pv),
                            len(a["pairs"] or []), a["arith"], a["row"], a["col"], a["cap"], a["ws"], a["ws_bytes"], None)
    return rc, lib.sce_last_error().decode()


@pytest.mark.parametrize("kw, msg", [
    (dict(a=None), "a is NULL"),
    (dict(na=0), "must be >= 1"),
    (dict(d=60), "multiple of 8"),
    (dict(d=16384), "8192"),
    (dict(a_norm=2), "normalize"),
    (dict(pairs=[]), "at least one pair"),
    (dict(pairs=[(2, 0)]), "outside"),
    (dict(pairs=[(0, -1)]), "outside"),
    (dict(b=1 << 23, mb=3, nb=32, pairs=[(0, 3)]), "outside"),
    (dict(b=1 << 23, mb=0, nb=32), "mb (0)"),
    (dict(a_rows=[64, 65]), "rows[1] of a = 65"),
    (dict(a_rows=[0, 64]), "rows[0] of a = 0"),
    (dict(b=1 << 23, mb=1, nb=32, b_rows=[33]), "rows[0] of b = 33"),
    (dict(arith=7), "unknown arith"),
    (dict(d=72, arith=_lib.SCE_ARITH_F16F8), "multiple of 16"),
    (dict(row=None, col=None), "no output"),
    (dict(b=1 << 23, mb=1, nb=32, cap=1 << 24), "self-pairs"),
    (dict(ws_bytes=1024), "workspace too small"),
    (dict(ws=(1 << 30) + 256), "1024-byte aligned"),
])
def test_similarity_abi_validation_without_device(kw, msg):
    rc, err = _call(_lib.load(), **kw)
    expect = -3 if "workspace" in msg or "aligned" in msg else -1   # SCE_ERR_WORKSPACE / SCE_ERR_INVALID
    assert rc == expect, (rc, err)
    assert msg in err, err


def test_similarity_workspace_bytes_rejects_bad_shapes():
    lib = _lib.load()
    assert lib.sce_similarity_workspace_bytes(0, 64, 0, 0, 64, 1, 0) == 0
    assert lib.sce_similarity_workspace_bytes(2, 64, 0, 0, 4, 1, 0) == 0
    assert lib.sce_similarity_workspace_bytes(2, 64, 0, 0, 64, 0, 0) == 0
    assert lib.sce_similarity_workspace_bytes(2, 64, 0, 0, 64, 1, 0) > 0


def test_similarity_workspace_at_config5_width():
    """Two 32768 x 2048 dictionaries, their pair and both self-pairs with capacity: operand planes (4 B per element)
    and O(P n ceil(n / 128)) partials, far below the 4 GiB one materialised [n, n] fp32 matrix would take."""
    lib = _lib.load()
    n, d = 32768, 2048
    ws = lib.sce_similarity_workspace_bytes(2, n, 0, 0, d, 3, 1)
    planes = 2 * n * d * 4
    partials = 3 * n * 2 * (n // 128) * 4 + 3 * n * 4
    assert planes + partials <= ws <= planes + partials + (1 << 20)
    assert ws < (4 << 30) // 4
    assert lib.sce_similarity_workspace_bytes(2, n, 0, 0, d, 1, 0) < planes + (1 << 20)   # no capacity: planes only


def _signatures():
    d, n, stack = 24, 40, 48
    torch.manual_seed(0)
    yield S.FunctionalTiedSAE, [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    yield S.FunctionalSAE, [S.FunctionalSAE.init(d, n, a) for a in (1e-3, 1e-2)]
    yield S.FunctionalMaskedTiedSAE, [S.FunctionalMaskedTiedSAE.init(d, k, stack, 1e-3) for k in (16, 48, 31)]
    yield S.FunctionalMaskedSAE, [S.FunctionalMaskedSAE.init(d, k, stack, 1e-3) for k in (16, 48, 31)]
    topk = [S.TopKEncoder.init(d, n, k) for k in (2, 5)]
    topk[0][0]["dict"][3] *= 1e-12                                   # tiny row: no clamp for TopK
    yield S.TopKEncoder, topk


@pytest.mark.parametrize("sig, models", list(_signatures()), ids=lambda x: getattr(x, "__name__", ""))
def test_learned_dict_stack_agrees_with_to_learned_dict(sig, models):
    params = stack_dict([p for p, _ in models])
    buffers = stack_dict([b for _, b in models])
    w, floor, rows = sig.learned_dict_stack(params, buffers)
    assert w.shape[0] == len(models)
    for m, (p, b) in enumerate(models):
        want = sig.to_learned_dict(p, b).get_learned_dict()
        k = int(rows[m]) if rows is not None else w.shape[1]
        got = w[m, :k]
        if floor is not None:
            nrm = got.norm(dim=-1)
            got = got / (nrm.clamp(min=floor) if floor > 0 else nrm)[:, None]
        assert got.shape == want.shape
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-7)


def test_similarity_needs_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        MT.mmcs(torch.randn(16, 8), torch.randn(8, 8))
