"""Synthetic datasets without a GPU: Philox4x32-10 against the Random123 known answers (numpy oracle and the torch
restatement the generators use), the numpy oracle of sce_synth_rows against a per-element brute force, the ground-truth
matrices against the reference's own (fixture), argument validation of the sce_synth_rows ABI, the per-group
probabilities, generator.pt pickling under the reference's names, and the chunk-file layout."""
import ctypes as C
import io
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import synth_oracle as O
from sparse_coding_b200 import _lib
from sparse_coding_b200 import synthetic as SY

KAT = [  # Random123 kat_vectors: philox4x32_10 (counter, key) -> output
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in O.philox4x32_10(*ctr, *key)) == want
    got = SY.philox4x32_10(*(torch.tensor(c) for c in ctr), key[0] | key[1] << 32)
    assert tuple(int(w) for w in got) == want


def test_torch_philox_matches_numpy_on_random_counters():
    rng = np.random.default_rng(3)
    c = rng.integers(0, 2 ** 32, size=(4, 1000), dtype=np.uint64)
    seed = int(rng.integers(0, 2 ** 63))
    want = O.philox4x32_10(*c, seed & 0xFFFFFFFF, seed >> 32)
    got = SY.philox4x32_10(*(torch.from_numpy(x.astype(np.int64)) for x in c), seed)
    for w, g in zip(want, got):
        assert np.array_equal(w.astype(np.int64), g.numpy())


def _philox_py(ctr, key):
    c, k = list(ctr), list(key)
    for _ in range(10):
        p0, p1 = O.M0 * c[0], O.M1 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
        k = [(k[0] + O.W0) & 0xFFFFFFFF, (k[1] + O.W1) & 0xFFFFFFFF]
    return c


def _u(x):
    return np.float32((x >> 8) * 2.0 ** -24)


@pytest.mark.parametrize("zero_rule,noise", [(True, 0.0), (False, 0.25)])
def test_oracle_matches_brute_force(zero_rule, noise):
    """The vectorised oracle against the contract of include/sce.h written out per draw."""
    rng = np.random.default_rng(0)
    n_gt, d, B, G, row0, seed = 11, 8, 12, 4, (1 << 32) - 5, 0x1234_5678_9ABC_DEF0
    feats = rng.standard_normal((n_gt, d)).astype(np.float32)
    probs = (rng.random((3, n_gt)) * 0.3).astype(np.float32)
    probs[1] = 0.0                                                        # rows 4..7: every row needs the zero-row rule
    probs[2, 3] = 1.5                                                     # always on
    lists, x = O.synth_rows(feats, probs, G, row0, B, seed, zero_rule, noise)
    key = (seed & 0xFFFFFFFF, seed >> 32)
    for i in range(B):
        r = row0 + i
        ctr = lambda q, tag: _philox_py((q, r & 0xFFFFFFFF, r >> 32, tag), key)
        idx, coef = [], []
        for j in range(n_gt):
            if _u(ctr(j // 4, 0)[j % 4]) <= probs[i // G, j]:
                idx.append(j)
                coef.append(_u(ctr(j // 4, 1)[j % 4]) * _u(ctr(j // 4, 2)[j % 4]))
        if not idx and zero_rule:
            j = (ctr(0, 3)[0] * n_gt) >> 32
            idx, coef = [j], [np.float32(1.0) * _u(ctr(j // 4, 2)[j % 4])]
        assert lists[i][0].tolist() == idx
        assert lists[i][1].tobytes() == np.array(coef, dtype=np.float32).tobytes()
        want = sum((np.float64(c) * feats[j].astype(np.float64) for j, c in zip(idx, coef)), np.zeros(d))
        for k in range(0, d, 4):
            w = ctr(k // 4, 4)
            for (a, b), col in (((w[0], w[1]), k), ((w[2], w[3]), k + 2)):
                rr = np.sqrt(-2 * np.log(((a >> 8) + 1) * 2.0 ** -24))
                t = 2 * np.pi * ((b >> 8) * 2.0 ** -24)
                want[col] += np.float32(noise) * rr * np.cos(t)
                want[col + 1] += np.float32(noise) * rr * np.sin(t)
        np.testing.assert_allclose(x[i], want, rtol=1e-12, atol=1e-12)
    assert all(len(lists[i][0]) == (1 if zero_rule else 0) for i in range(4, 8))
    assert all(3 in lists[i][0] for i in range(8, 12))


def test_ground_truth_matrices_match_the_reference(golden):
    g = golden("synthetic")
    np.random.seed(g["config"]["np_seed"])
    feats = SY.generate_rand_feats(g["config"]["d"], g["config"]["n_gt"], "cpu")
    corr = SY.generate_corr_matrix(g["config"]["n_gt"], "cpu")
    assert feats.dtype == corr.dtype == torch.float32
    assert (feats - g["feats"]).abs().max() <= 1e-6 and (corr - g["corr"]).abs().max() <= 1e-6
    np.random.seed(g["config"]["np_seed"])                                # the generators draw them the same way
    gen = SY.SparseMixDataset(64, 128, 4096, 5, 0.99, 0.1, "cpu", seed=7)
    assert torch.equal(gen.sparse_component_dict, feats) and torch.equal(gen.sparse_component_covariance, corr)
    np.random.seed(g["config"]["np_seed"])
    rgen = SY.RandomDatasetGenerator(64, 128, 4096, 5, 0.99, False, "cpu", seed=7)
    assert torch.equal(rgen.feats, feats) and rgen.corr_matrix is None


def _synth(lib, **kw):
    a = dict(feats=1 << 20, n_gt=16, d=64, probs=1 << 21, group_rows=8, row0=0, B=32, seed=1, zero=1, noise=0.0,
             out=1 << 22, half=0, nnz=None, idx=None, val=None, cap=0)
    a.update(kw)
    rc = lib.sce_synth_rows(a["feats"], a["n_gt"], a["d"], a["probs"], a["group_rows"], a["row0"], a["B"], a["seed"],
                            a["zero"], C.c_float(a["noise"]), a["out"], a["half"], a["nnz"], a["idx"], a["val"],
                            a["cap"], None)
    return rc, lib.sce_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    ({"feats": None}, "required"), ({"probs": None}, "required"), ({"out": None}, "required"),
    ({"n_gt": 0}, "n_gt"), ({"B": 0}, "B (0)"), ({"d": 12}, "multiple of 8"), ({"d": 0}, "multiple of 8"),
    ({"d": 8200}, "8192"), ({"group_rows": 0}, "group_rows"), ({"row0": -1}, "row0"), ({"zero": 2}, "0 or 1"),
    ({"half": 3}, "0 or 1"), ({"noise": -1.0}, "noise_scale"), ({"noise": float("nan")}, "noise_scale"),
    ({"noise": float("inf")}, "noise_scale"), ({"idx": 1 << 23}, "together"), ({"val": 1 << 23}, "together"),
    ({"idx": 1 << 23, "val": 1 << 24, "cap": 0}, "code_cap"), ({"out": (1 << 22) + 8}, "16-byte"),
    ({"feats": (1 << 20) + 4}, "16-byte"),
])
def test_synth_rows_validation_without_device(kw, msg):
    rc, err = _synth(_lib.load(), **kw)
    assert rc == -1 and msg in err, (kw, err)


def test_group_probabilities():
    """generate_correlated_dataset's probabilities: mean frac_nonzero per group (nothing clipped), the Gaussians of the
    kernel's contract, the covariance through its Cholesky factor, and one draw per group (rows of a group share it)."""
    np.random.seed(1)
    gen = SY.SparseMixDataset(32, 96, 64, 6, 0.98, 0.0, "cpu", seed=5)
    p = gen._group_probs(0, 5)
    assert p.shape == (5, 96) and p.dtype == torch.float32
    torch.testing.assert_close(p.double().mean(1), torch.full((5,), 6 / 96, dtype=torch.float64), rtol=1e-6, atol=0)
    assert not torch.equal(p[0], p[1])
    torch.testing.assert_close(gen._group_probs(3, 1)[0], p[3])           # a group's draw depends on its index only
    z = torch.from_numpy(O.group_gaussians(5, np.arange(5), 96))
    torch.testing.assert_close(SY.group_gaussians(5, 0, 5, 96, "cpu").double(), z, rtol=0, atol=1e-5)
    L = torch.linalg.cholesky(gen.sparse_component_covariance.double())
    want = torch.special.ndtr(z @ L.T) * gen.sparse_component_probs.double()
    want = want * (6 / 96 / want.mean(1, keepdim=True))
    torch.testing.assert_close(p.double(), want, rtol=1e-4, atol=1e-6)
    eye = SY.SparseMixDataset(32, 96, 64, 6, 0.98, 0.0, "cpu", sparse_component_covariance=torch.eye(96), seed=5)
    want = torch.special.ndtr(z) * eye.sparse_component_probs.double()
    torch.testing.assert_close(eye._group_probs(0, 5).double(), want * (6 / 96 / want.mean(1, keepdim=True)),
                               rtol=1e-5, atol=1e-7)
    rgen = SY.RandomDatasetGenerator(32, 96, 64, 6, 0.98, False, "cpu", seed=5)
    assert torch.equal(rgen._group_probs(0, 2)[1], (rgen.decay * (6 / 96)).float())


def test_noise_covariance_must_be_the_identity():
    with pytest.raises(NotImplementedError):
        SY.SparseMixDataset(8, 16, 4, 2, 1.0, 0.1, "cpu", noise_covariance=2 * torch.eye(8), seed=1)
    with pytest.raises(NotImplementedError):
        SY.generate_noise_dataset(4, 2 * torch.eye(8), 0.1, "cpu")


def test_seed_comes_from_torch_default_generator():
    torch.manual_seed(123)
    a = SY.SparseMixDataset(8, 16, 4, 2, 1.0, 0.0, "cpu").seed
    torch.manual_seed(123)
    b = SY.SparseMixDataset(8, 16, 4, 2, 1.0, 0.0, "cpu").seed
    assert a == b and 0 <= a < 2 ** 63


def test_generator_pickles_under_reference_names(tmp_path):
    np.random.seed(0)
    gen = SY.SparseMixDataset(16, 24, 8, 3, 0.99, 0.1, "cpu", torch.randn(24, 16), torch.eye(24), t_type=torch.float16,
                              seed=99)
    gen._group_probs(0, 1)                                                # builds the cached factor
    gen._group, gen._row = 3, 24
    raw = pickle.dumps(gen)
    assert b"sc_datasets.random_dataset" in raw and b"SparseMixDataset" in raw and b"_chol_cache" not in raw
    path = tmp_path / "generator.pt"
    torch.save(gen, path)
    back = torch.load(path, weights_only=False)
    assert type(back) is SY.SparseMixDataset and type(back).__module__ == "sc_datasets.random_dataset"
    assert torch.equal(back.sparse_component_dict, gen.sparse_component_dict) and back.t_type == torch.float16
    assert (back.seed, back._group, back._row) == (99, 3, 24)
    assert torch.equal(back._group_probs(0, 2), gen._group_probs(0, 2))
    # a generator.pt written by the reference carries the dataclass fields only: it loads and starts a stream
    state = {k: v for k, v in gen.__dict__.items() if k not in ("seed", "_group", "_row", "_chol_cache")}
    ref_like = SY.SparseMixDataset.__new__(SY.SparseMixDataset)
    ref_like.__dict__.update(state)
    buf = io.BytesIO()
    pickle.Pickler(buf).dump(ref_like.__dict__)
    obj = SY.SparseMixDataset.__new__(SY.SparseMixDataset)
    obj.__setstate__(pickle.loads(buf.getvalue()))
    assert isinstance(obj.seed, int) and (obj._group, obj._row) == (0, 0)
    assert obj.sparse_component_dict.shape == (24, 16)
    rgen = SY.RandomDatasetGenerator(8, 12, 4, 2, 1.0, True, "cpu", seed=3)
    assert b"sc_datasets.random_dataset" in pickle.dumps(rgen)


@pytest.mark.parametrize("correlated", [False, True])
def test_random_generator_zero_row_rule_follows_its_path(correlated):
    """generate_rand_dataset has no zero-row rule, generate_correlated_dataset has one: the generator applies the rule of
    its path, also when loaded from a pickle that holds only the reference's fields."""
    rgen = SY.RandomDatasetGenerator(8, 12, 4, 2, 1.0, correlated, "cpu", seed=3)
    assert rgen._zero_row_rule is correlated
    assert pickle.loads(pickle.dumps(rgen))._zero_row_rule is correlated
    fields = {k: v for k, v in rgen.__dict__.items() if not k.startswith("_") and k != "seed"}
    obj = SY.RandomDatasetGenerator.__new__(SY.RandomDatasetGenerator)
    obj.__setstate__(pickle.loads(pickle.dumps(fields)))
    assert obj._zero_row_rule is correlated and isinstance(obj.seed, int)


class _FakeGenerator:
    """sends(n) -> n sends of 3 rows; values that fp16 rounds."""
    batch_size = 3

    def __init__(self):
        self.n = 0

    def sends(self, n):
        x = (torch.arange(n * 3 * 8, dtype=torch.float64).reshape(n * 3, 8) + self.n + 1 / 3).half()
        self.n += n * 3 * 8
        return x


def test_chunk_file_layout(tmp_path):
    assert SY.chunk_rows_for(512, 2.0) == 2 ** 21 and SY.chunk_rows_for(512, 2) == 2 ** 21
    assert SY.chunk_rows_for(768, 0.5) == 349525
    cfg = type("Cfg", (), {"dataset_folder": str(tmp_path), "activation_width": 8})()
    gen = _FakeGenerator()
    SY.generate_synthetic_dataset(cfg, gen, 10, 2)
    assert sorted(os.listdir(tmp_path)) == ["0.pt", "1.pt"]
    ref = _FakeGenerator()
    for i in range(2):
        c = torch.load(tmp_path / f"{i}.pt")
        assert c.dtype == torch.float32 and c.shape == (10, 8)
        assert torch.equal(c[:9], ref.sends(3).float())                   # 3 whole sends, fp16 values held in fp32
        assert torch.equal(c[9:], torch.zeros(1, 8))                      # the rows past the last full send


def test_synthetic_chunks_order_and_bounds():
    gen = SY.SparseMixDataset(8, 16, 4, 2, 1.0, 0.0, "cpu", seed=1)
    sc = SY.SyntheticChunks(gen, 3, 16, order=[2, 0, 2])
    assert len(sc) == 3 and sc.order == [2, 0, 2] and len(SY.SyntheticChunks(gen, 3, 16)) == 3
    with pytest.raises(ValueError):
        SY.SyntheticChunks(gen, 3, 16, order=[3])
    with pytest.raises(ValueError):
        SY.SyntheticChunks(gen, 3, 2)
    with pytest.raises(RuntimeError):                                     # the rows come from the CUDA engine only
        gen.send(None)
