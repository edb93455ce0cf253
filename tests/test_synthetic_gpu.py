"""Synthetic datasets on the GPU: sce_synth_rows against the numpy oracle (active lists and coefficients bitwise, fp32
rows to the rounding of fp32 FMAs, fp16 rows to the correctly rounded value), independence from how rows are split
over calls, the chunks, the reference's statistics (tests/golden/synthetic.pt), and ground-truth recovery by
training on generated chunks."""
import os

import numpy as np
import pytest
import torch

from oracle import synth_oracle as O
from sparse_coding_b200 import synthetic as SY

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _case(d, n_gt, B=96, G=16, nnz=12, seed=0x5EED_0000_0001):
    rng = np.random.default_rng(d + n_gt)
    feats = rng.standard_normal((n_gt, d)).astype(np.float32)
    feats /= np.linalg.norm(feats, axis=1, keepdims=True)
    groups = (B + G - 1) // G
    probs = (rng.random((groups, n_gt)) * (2.0 * nnz / n_gt)).astype(np.float32)
    probs[1] = 0.0                                       # a group of empty rows: the zero-row rule decides them
    probs[2, :3] = 1.25                                  # always on
    return feats, probs, G, (1 << 32) - 40, B, seed


def _run(feats, probs, G, row0, B, seed, zero, noise, dtype, cap):
    return SY.synth_rows(torch.from_numpy(feats).to(DEV), torch.from_numpy(probs).to(DEV), G, row0, B, seed, zero,
                         noise, dtype, code_cap=cap)


def _check_lists(lists, nnz, idx, val, cap):
    nnz, idx, val = nnz.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()
    for i, (li, lv) in enumerate(lists):
        assert nnz[i] == len(li), i
        k = min(len(li), cap)
        assert np.array_equal(idx[i, :k], li[:k]), i
        assert val[i, :k].tobytes() == lv[:k].tobytes(), i


@pytest.mark.parametrize("d,n_gt", [(64, 128), (512, 2048), (2048, 4096), (8192, 512)])
@pytest.mark.parametrize("zero,noise", [(True, 0.1), (False, 0.0)])
def test_rows_match_oracle(d, n_gt, zero, noise):
    feats, probs, G, row0, B, seed = _case(d, n_gt)
    lists, x64 = O.synth_rows(feats, probs, G, row0, B, seed, zero, noise)
    z = O.noise(seed, row0 + np.arange(B), d) if noise else np.zeros((B, d))
    coef_abs = np.array([np.abs(lv.astype(np.float64)).sum() for _, lv in lists])
    # fp32: the FMA chain of at most n_gt terms, |feats| <= 1, plus the fp32 Box-Muller (a few ulp of noise * z)
    tol = 1e-6 * (coef_abs[:, None] + np.float32(noise) * np.abs(z))
    x, nnz, idx, val = _run(feats, probs, G, row0, B, seed, zero, noise, torch.float32, n_gt)
    _check_lists(lists, nnz, idx, val, n_gt)
    err = np.abs(x.cpu().numpy().astype(np.float64) - x64)
    assert (err <= tol).all(), float((err / tol).max())
    assert (nnz.cpu().numpy()[16:32] == (1 if zero else 0)).all()
    # fp16: the fp64 value rounded to nearest; one ulp apart only where it lies within tol of a rounding boundary
    h, nnz16, idx16, val16 = _run(feats, probs, G, row0, B, seed, zero, noise, torch.float16, 4)
    _check_lists(lists, nnz16, idx16, val16, 4)                              # lists truncated at code_cap
    h = h.cpu().numpy()
    rn = x64.astype(np.float16)
    off = h != rn
    if off.any():
        hv, rv, xv, tv = h[off].astype(np.float64), rn[off].astype(np.float64), x64[off], tol[off]
        ulp = np.abs(np.spacing(rn[off]).astype(np.float64))
        assert (np.abs(hv - rv) <= ulp * 1.0001).all()
        assert (np.abs(xv - (hv + rv) / 2) <= tv).all()


@pytest.mark.parametrize("d,n_gt", [(512, 2048), (2048, 2048), (8192, 1024)])
def test_dense_rows_match_oracle(d, n_gt):
    """Rows with far more active components than the kernel's 256-entry shared list, so that it is gathered and reset
    several times within a row (in the warp-per-row kernel at d = 512, in the block-per-row kernel above 1024, where
    the count is handed to the other warps through shared memory). Groups of 16 rows: p = 0.3 (~0.3 n_gt active),
    p = 0 (zero-row rule), p = 1/16 at n_gt = 2048 (~128 active, around the flush bound), p = 1 (every component)."""
    rng = np.random.default_rng(d)
    feats = rng.standard_normal((n_gt, d)).astype(np.float32)
    feats /= np.linalg.norm(feats, axis=1, keepdims=True)
    G, B, row0, seed = 16, 80, (1 << 33) + 7, 0xD15E_A5E0_0002
    dens = [0.3, 0.0, 128.0 / n_gt, 1.0, 0.3]
    probs = np.stack([np.full(n_gt, p, dtype=np.float32) * (0.9 + 0.2 * rng.random(n_gt, dtype=np.float32))
                      for p in dens]).astype(np.float32)
    probs[3] = 1.0
    for zero, noise in ((True, 0.1), (False, 0.0)):
        lists, x64 = O.synth_rows(feats, probs, G, row0, B, seed, zero, noise)
        counts = np.array([len(li) for li, _ in lists])
        assert counts[:16].min() > 256 and (counts[48:64] == n_gt).all()                    # several flushes per row
        z = O.noise(seed, row0 + np.arange(B), d) if noise else np.zeros((B, d))
        coef_abs = np.array([np.abs(lv.astype(np.float64)).sum() for _, lv in lists])
        tol = 1e-6 * (coef_abs[:, None] + np.float32(noise) * np.abs(z))
        for cap in (n_gt, 200):                                                               # lists uncapped and capped
            x, nnz, idx, val = _run(feats, probs, G, row0, B, seed, zero, noise, torch.float32, cap)
            _check_lists(lists, nnz, idx, val, cap)
            err = np.abs(x.cpu().numpy().astype(np.float64) - x64)
            assert (err <= tol).all(), (cap, float((err / tol).max()))


def _valid(nnz, idx, val):
    """The list entries a call defines (those below min(row_nnz, code_cap)); the rest of the buffers are not written."""
    keep = torch.arange(idx.shape[1], device=idx.device)[None, :] < nnz[:, None]
    return torch.where(keep, idx, -1), torch.where(keep, val, -1.0)


def test_rows_do_not_depend_on_the_split_or_the_run():
    feats, probs, G, row0, B, seed = _case(512, 2048, B=256)
    x, nnz, idx, val = _run(feats, probs, G, row0, B, seed, True, 0.1, torch.float32, 64)
    x2, nnz2, idx2, val2 = _run(feats, probs, G, row0, B, seed, True, 0.1, torch.float32, 64)
    lists = _valid(nnz, idx, val)
    assert torch.equal(x, x2) and torch.equal(nnz, nnz2)
    assert all(torch.equal(a, b) for a, b in zip(lists, _valid(nnz2, idx2, val2)))
    parts = []
    for lo, hi in ((0, 48), (48, 160), (160, 256)):                         # group-aligned pieces, each its own row0
        parts.append(_run(feats, probs[lo // G:], G, row0 + lo, hi - lo, seed, True, 0.1, torch.float32, 64))
    assert torch.equal(torch.cat([p[0] for p in parts]), x)
    assert torch.equal(torch.cat([p[1] for p in parts]), nnz)
    split = _valid(nnz, torch.cat([p[2] for p in parts]), torch.cat([p[3] for p in parts]))
    assert all(torch.equal(a, b) for a, b in zip(lists, split))


def test_sends_chunks_and_files_agree(tmp_path):
    np.random.seed(4)
    mk = lambda: SY.SparseMixDataset(128, 256, 512, 6, 0.99, 0.1, "cuda", seed=17,
                                     sparse_component_covariance=None, t_type=torch.float16)
    gen = mk()
    sends = torch.cat([gen.send(None) for _ in range(5)])
    assert sends.dtype == torch.float16 and sends.shape == (2560, 128)
    np.random.seed(4)
    gen2 = mk()
    assert torch.equal(gen2.sends(5), sends)                                   # n sends == one call of n groups
    np.random.seed(4)
    gen3 = mk()
    chunks = SY.SyntheticChunks(gen3, 3, 2300, order=[1, 0, 1])
    got = list(chunks)
    assert [i for i, _ in got] == [1, 0, 1] and torch.equal(got[0][1], got[2][1])   # regenerated bitwise
    c0 = got[1][1]
    assert c0.shape == (2300, 128) and torch.equal(c0[:2048], sends[:2048]) and not c0[2048:].any()
    np.random.seed(4)
    gen4 = mk()
    cfg = type("Cfg", (), {"dataset_folder": str(tmp_path), "activation_width": 128})()
    SY.generate_synthetic_dataset(cfg, gen4, 2300, 2)
    assert torch.equal(torch.load(tmp_path / "0.pt"), c0.float().cpu())
    assert torch.equal(torch.load(tmp_path / "1.pt"), got[0][1].float().cpu())


def test_reference_functions_return_codes():
    np.random.seed(0)
    feats = SY.generate_rand_feats(64, 96, DEV)
    torch.manual_seed(0)
    probs = torch.full((96,), 0.02, device=DEV)
    f, codes, x = SY.generate_rand_dataset(96, 500, probs, feats, DEV)
    assert f is feats and codes.shape == (500, 96) and x.shape == (500, 64)
    assert ((codes >= 0) & (codes < 1)).all() and (codes.count_nonzero(1) == 0).any()   # no zero-row rule here
    decay = torch.ones(96, device=DEV)
    _, codes, x = SY.generate_correlated_dataset(96, 500, torch.eye(96, device=DEV), feats, 0.01, decay, DEV)
    assert (codes.count_nonzero(1) >= 1).all() and (codes == 1.0).any()      # zero rows filled with a 1.0
    n = SY.generate_noise_dataset(4096, torch.eye(64, device=DEV), 0.1, DEV)
    assert n.shape == (4096, 64) and abs(float(n.var()) - 0.01) < 5e-4 and abs(float(n.mean())) < 1e-3


def _stats(gen, corr, noise, sends):
    """Per-send statistics as oracle/make_synth_golden.py records them for the reference."""
    bs = gen.batch_size
    feats = gen._feats()
    n_gt = feats.shape[0]
    per = []
    for g in range(sends):
        p = gen._group_probs(g, 1)
        x, nnz, idx, val = SY.synth_rows(feats, p, bs, g * bs, bs, gen.seed, corr, noise, code_cap=n_gt)
        codes = SY._dense_codes(gen.seed, g * bs, nnz, idx, val, p if corr else None, n_gt)
        keep = torch.arange(n_gt, device=DEV)[None, :] < nnz[:, None]
        coef = val[keep].double()
        nzc = (codes != 0).sum(1)
        K = 16
        hist = torch.stack([(nzc == k).double().mean() for k in range(K - 1)] + [(nzc >= K - 1).double().mean()])
        norm = x.double().norm(dim=1)
        s = {"freq": (codes != 0).double().mean(0), "nnz_hist": hist, "fill": (codes == 1.0).any(1).double().mean(),
             "coef_mean": coef.mean(), "coef_var": coef.var(), "norm_mean": norm.mean(), "norm_var": norm.var()}
        if noise:
            clean, _, _, _ = SY.synth_rows(feats, p, bs, g * bs, bs, gen.seed, corr, 0.0)
            s["noise_var"] = (x - clean).double().var()
        per.append({k: v.cpu() for k, v in s.items()})
    return {k: torch.stack([s[k] for s in per]) for k in per[0]}


@pytest.mark.parametrize("which", ["sparse_mix", "random"])
def test_statistics_match_the_reference(golden, which):
    """Each statistic's mean over sends within 5 sigma of the reference's, sigma = the standard error of the difference
    of the two means, sqrt(var_ref / S + var_ours / S), each variance taken over the S independent sends (plus 1e-12
    for statistics that never vary)."""
    g = golden("synthetic")
    c = g["config"]
    np.random.seed(c["np_seed"])
    if which == "sparse_mix":
        gen = SY.SparseMixDataset(c["d"], c["n_gt"], c["batch"], c["nnz"], c["decay"], c["noise"], "cuda", seed=11)
        ours = _stats(gen, True, c["noise"], c["sends"])
    else:
        gen = SY.RandomDatasetGenerator(c["d"], c["n_gt"], c["batch"], c["nnz"], c["decay"], False, "cuda", seed=11)
        ours = _stats(gen, False, 0.0, c["sends"])
    ref = g[which]
    assert set(ours) == set(ref)
    for k in ref:
        a, b = ref[k].double(), ours[k].double()
        S = a.shape[0]
        sigma = torch.sqrt(a.var(0) / S + b.var(0) / S) + 1e-12
        z = (a.mean(0) - b.mean(0)).abs() / sigma
        assert (z <= 5).all(), (which, k, float(z.max()), a.mean(0), b.mean(0))
    if which == "sparse_mix":
        assert 0 < float(ours["fill"].mean()) < 0.05                         # the zero-row rule fires, rarely


def _ld_mmcs(encoders, truth):
    import sparse_coding_b200 as S
    return [float(S.metrics.mmcs_to_fixed(S.TiedSAE(e, torch.zeros(e.shape[0], device=DEV)), truth)) for e in encoders]


def test_ground_truth_recovery(tmp_path):
    """Tied SAEs trained on generated chunks find the generator's features: the best of eight L1 values reaches a mean
    max cosine of 0.9 to the ground truth; the engine and the PyTorch oracle step agree on it within 0.02."""
    import sparse_coding_b200 as S
    from oracle import sae_oracle as RO
    from sparse_coding_b200.train_loop import train_on_chunks
    d, n_gt, nnz, bs = 256, 512, 5, 1024
    np.random.seed(0)
    gen = S.SparseMixDataset(d, n_gt, 4096, nnz, 1.0, 0.0, "cuda", sparse_component_covariance=torch.eye(n_gt),
                             t_type=torch.float16, seed=2024)
    truth = gen.sparse_component_dict
    torch.manual_seed(0)
    l1 = np.logspace(-4, -2, 8)
    models = [S.FunctionalTiedSAE.init(d, n_gt, float(a)) for a in l1]
    clone = lambda dev: [({k: v.clone().to(dev) for k, v in p.items()}, {k: v.clone().to(dev) for k, v in b.items()})
                         for p, b in models]
    ens = S.FunctionalEnsemble(clone("cpu"), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    chunks = S.SyntheticChunks(gen, 4, 1 << 19)
    dicts = train_on_chunks(ens, {"device": "cuda"}, None, str(tmp_path / "out"), bs, [], ["l1_alpha"], chunks=chunks)
    assert len(dicts) == 8 and os.path.exists(tmp_path / "out" / "_3" / "learned_dicts.pt")
    mmcs = []
    for ld, _ in dicts:
        ld.to_device(DEV)
        mmcs.append(float(S.metrics.mmcs_to_fixed(ld, truth)))
    assert max(mmcs) >= 0.9, mmcs

    # the same 256 batches of one generated chunk through the engine and the oracle step
    chunk = chunks.chunk(0).float()
    ens2 = S.FunctionalEnsemble(clone("cpu"), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device=DEV)
    ref = RO.RefPortEnsemble(clone(DEV), RO.SIG_LOSSES["tied"], lr=1e-3)
    perm = torch.randperm(chunk.shape[0], generator=torch.Generator().manual_seed(0)).to(DEV)
    for s in range(256):
        batch = chunk[perm[s * bs:(s + 1) * bs]]
        ens2.step_batch(batch)
        ref.step_batch(batch)
    a = _ld_mmcs(list(ens2.params["encoder"]), truth)
    b = _ld_mmcs(list(ref.params["encoder"]), truth)
    assert max(abs(x - y) for x, y in zip(a, b)) <= 0.02, (a, b)
