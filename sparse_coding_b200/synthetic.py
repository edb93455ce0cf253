"""Synthetic sparse-mixture datasets with a known ground truth, generated on the GPU (sc_datasets/random_dataset.py).

The reference's synthetic sweep (big_sweep.py:228-237, 269-295) builds a ``SparseMixDataset``, writes ``n_chunks``
activation chunks from it and pickles the generator to ``generator.pt``, whose ``sparse_component_dict`` the plotting
scripts score every learned dictionary against (``mmcs_to_fixed``). This module provides the same classes, functions
and files with the rows made by libsce ``sce_synth_rows``: per row, the active components are found by thresholds
drawn from a counter-based generator (Philox4x32-10, include/sce.h), and ``x`` is gathered from the active feature
rows only, so the dense [rows, n_gt] code, its three uniform tensors and the fp32 GEMM are never formed.

What follows the reference exactly: the ground-truth matrices (``generate_rand_feats`` and ``generate_corr_matrix``
draw from numpy's global generator in the same way and order, so ``np.random.seed`` gives the reference's
``sparse_component_dict``), the distributions (one correlated Gaussian vector per send, ``p = ndtr(z) decay`` scaled
to mean ``frac_nonzero``, ``u_thresh <= p``, coefficient ``u_val u_strength``, the zero-row rule of
generate_correlated_dataset, identity noise), the chunk files, and the pickled class names. The random streams are
not torch's: a row is a pure function of (seed, global row, probabilities), whichever call or GPU produced it.

``SyntheticChunks`` hands the chunks straight to ``train_on_chunks(chunks=...)``: each GPU generates its chunk in HBM,
with no file, no broadcast and no PCIe traffic, and a repeated chunk is regenerated bitwise."""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Any, Generator, Iterable, Optional, Tuple, Union

import numpy as np
import torch

from . import _lib

_REF_MODULE = "sc_datasets.random_dataset"

# Philox4x32-10 stream tags (include/sce.h); the per-group Gaussians use the tag the kernel leaves to its caller
TAG_THRESH, TAG_VALUE, TAG_STRENGTH, TAG_ZERO, TAG_NOISE, TAG_GAUSS = range(6)
_M0, _M1, _W0, _W1, _MASK = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF


# ----------------------------------------------------------------------------------------------------------------
# ground-truth matrices: numpy's global generator, as random_dataset.py:248-279
# ----------------------------------------------------------------------------------------------------------------
def generate_rand_feats(feat_dim: int, num_feats: int, device) -> torch.Tensor:
    """[num_feats, feat_dim] fp32: rows of ``np.random.multivariate_normal(0, I)``, unit-normalised."""
    feats = np.random.multivariate_normal(np.zeros(feat_dim), np.eye(feat_dim), size=num_feats)
    feats = feats.T / np.linalg.norm(feats, axis=1)
    return torch.from_numpy(feats.T).to(device).float()


def generate_corr_matrix(num_feats: int, device) -> torch.Tensor:
    """[num_feats, num_feats] fp32: ``np.random.rand`` symmetrised, shifted by 1.001 |min eig| when that is negative."""
    corr_matrix = np.random.rand(num_feats, num_feats)
    corr_matrix = (corr_matrix + corr_matrix.T) / 2
    min_eig = np.min(np.real(np.linalg.eigvals(corr_matrix)))
    if min_eig < 0:
        corr_matrix -= 1.001 * min_eig * np.eye(corr_matrix.shape[0], corr_matrix.shape[1])
    return torch.from_numpy(corr_matrix).to(device).float()


# ----------------------------------------------------------------------------------------------------------------
# the kernel's random numbers, restated in torch (int64 lanes holding uint32) for the few draws made outside it
# ----------------------------------------------------------------------------------------------------------------
def _mulhilo(m: int, c: torch.Tensor):
    """(hi, lo) 32-bit words of m * c for a uint32 constant m and uint32 values c, without 64-bit overflow."""
    t = c * (m & 0xFFFF)
    u = c * (m >> 16)
    return (u + (t >> 16)) >> 16, (((u & 0xFFFF) << 16) + t) & _MASK


def philox4x32_10(c0, c1, c2, c3, seed: int):
    """Philox4x32-10 of the counter (c0, c1, c2, c3) (int64 tensors of uint32 values, broadcast) under key ``seed``."""
    k0, k1 = seed & _MASK, (seed >> 32) & _MASK
    dev = next((c.device for c in (c0, c1, c2, c3) if torch.is_tensor(c)), None)
    c0, c1, c2, c3 = torch.broadcast_tensors(*(torch.as_tensor(c, dtype=torch.int64, device=dev)
                                               for c in (c0, c1, c2, c3)))
    for _ in range(10):
        hi0, lo0 = _mulhilo(_M0, c0)
        hi1, lo1 = _mulhilo(_M1, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return c0, c1, c2, c3


def _uniform(x: torch.Tensor) -> torch.Tensor:
    return (x >> 8).float() * 2.0 ** -24


def group_gaussians(seed: int, group0: int, n_groups: int, n: int, device) -> torch.Tensor:
    """[n_groups, n] fp32 standard normals of groups group0 .. group0 + n_groups - 1: Philox counter
    (k / 4, group lo, group hi, TAG_GAUSS), Box-Muller on the word pairs as the kernel's noise (include/sce.h)."""
    g = torch.arange(group0, group0 + n_groups, dtype=torch.int64, device=device)[:, None]
    q = torch.arange((n + 3) // 4, dtype=torch.int64, device=device)[None, :]
    w = philox4x32_10(q, g & _MASK, g >> 32, TAG_GAUSS, seed)
    z = []
    for a, b in ((w[0], w[1]), (w[2], w[3])):
        r = torch.sqrt(-2.0 * torch.log(((a >> 8) + 1).float() * 2.0 ** -24))
        ang = (2.0 * math.pi) * _uniform(b)
        z += [r * torch.cos(ang), r * torch.sin(ang)]
    return torch.stack(z, dim=-1).reshape(n_groups, -1)[:, :n].contiguous()


def _draw_seed() -> int:
    """One 63-bit draw from torch's default generator, so ``torch.manual_seed`` governs a run as in the reference."""
    return int(torch.empty((), dtype=torch.int64).random_().item())


def _is_identity(c: torch.Tensor) -> bool:
    return c.dim() == 2 and c.shape[0] == c.shape[1] and torch.equal(c, torch.eye(c.shape[0], dtype=c.dtype, device=c.device))


def _cholesky(cov: torch.Tensor) -> Optional[torch.Tensor]:
    """The factor MultivariateNormal(covariance_matrix=cov) samples with, or None for the identity."""
    return None if _is_identity(cov) else torch.linalg.cholesky(cov.float())


def component_probs(z: torch.Tensor, chol: Optional[torch.Tensor], decay: torch.Tensor, frac_nonzero: float):
    """generate_correlated_dataset's probabilities (random_dataset.py:213-226) of each row of standard normals z
    [G, n]: p = ndtr(z L^T) decay, scaled to mean frac_nonzero; a p > 1 is left as is (always on). fp32, TF32 off."""
    if chol is not None:
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            z = z @ chol.T
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
    p = torch.special.ndtr(z) * decay
    return p * (frac_nonzero / p.mean(dim=-1, keepdim=True))


# ----------------------------------------------------------------------------------------------------------------
# the kernel
# ----------------------------------------------------------------------------------------------------------------
def synth_rows(feats: torch.Tensor, probs: torch.Tensor, group_rows: int, row0: int, B: int, seed: int,
               zero_row_rule: bool, noise_scale: float, out_dtype=torch.float32, code_cap: int = 0,
               out: Optional[torch.Tensor] = None):
    """libsce sce_synth_rows: (x [B, d] fp32 or fp16, row_nnz [B] int32, code_idx, code_val [B, code_cap] or None)."""
    if not feats.is_cuda:
        raise RuntimeError("synthetic rows are generated by the CUDA engine; the generator must live on a GPU")
    if out_dtype not in (torch.float32, torch.float16):
        raise TypeError("the kernel writes fp32 or fp16 rows")
    feats = feats.float().contiguous()
    probs = probs.to(device=feats.device, dtype=torch.float32).contiguous()
    n_gt, d = feats.shape
    dev = feats.device
    if out is None:
        out = torch.empty(B, d, dtype=out_dtype, device=dev)
    assert out.shape == (B, d) and out.dtype == out_dtype and out.is_contiguous()
    nnz = torch.empty(B, dtype=torch.int32, device=dev)
    idx = val = None
    if code_cap:
        idx = torch.empty(B, code_cap, dtype=torch.int32, device=dev)
        val = torch.empty(B, code_cap, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(_lib.load().sce_synth_rows(
            feats.data_ptr(), n_gt, d, probs.data_ptr(), group_rows, row0, B, seed & 0xFFFFFFFFFFFFFFFF,
            int(bool(zero_row_rule)), float(noise_scale), out.data_ptr(), int(out_dtype == torch.float16),
            nnz.data_ptr(), idx.data_ptr() if idx is not None else None, val.data_ptr() if val is not None else None,
            code_cap, stream), "sce_synth_rows")
    return out, nnz, idx, val


def _dense_codes(seed: int, row0: int, nnz, idx, val, probs: Optional[torch.Tensor], n_gt: int) -> torch.Tensor:
    """The reference's ``dataset_codes`` [B, n_gt]: u_val where a component is active, 1.0 where the zero-row rule
    filled the row (``probs`` given: an entry whose threshold fails is such a fill), 0 elsewhere."""
    B, cap = idx.shape
    keep = torch.arange(cap, device=idx.device)[None, :] < nnz[:, None]
    r, k = keep.nonzero(as_tuple=True)
    j = idx[r, k].long()
    grow = r.long() + row0
    q, lo, hi = j >> 2, grow & _MASK, grow >> 32
    pick = lambda w: torch.stack(w, -1).gather(-1, (j & 3)[:, None])[:, 0]
    code = _uniform(pick(philox4x32_10(q, lo, hi, TAG_VALUE, seed)))
    if probs is not None:
        fill = _uniform(pick(philox4x32_10(q, lo, hi, TAG_THRESH, seed))) > probs.reshape(-1)[j]
        code = torch.where(fill, torch.ones_like(code), code)
    codes = torch.zeros(B, n_gt, dtype=torch.float32, device=idx.device)
    codes[r, j] = code
    return codes


def generate_noise_dataset(dataset_size: int, noise_covariance: torch.Tensor, noise_magnitude_scale: float,
                           device) -> torch.Tensor:
    """random_dataset.py:145-157: [dataset_size, d] fp32 noise_magnitude_scale * N(0, I), drawn by sce_synth_rows
    (its noise stream), so d must be a multiple of 8 in [8, 8192] as for every generated row; other widths raise."""
    if not _is_identity(noise_covariance):
        raise NotImplementedError("only the identity noise covariance is generated (the one every caller uses)")
    d = noise_covariance.shape[0]
    zeros = torch.zeros(1, d, device=device)
    x, _, _, _ = synth_rows(zeros, torch.zeros(1, 1, device=device), dataset_size, 0, dataset_size, _draw_seed(),
                            False, noise_magnitude_scale)
    return x


def generate_rand_dataset(n_ground_truth_components: int, dataset_size: int, feature_probs: torch.Tensor,
                          feats: torch.Tensor, device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """random_dataset.py:160-188: fixed probabilities, no zero-row rule, no noise. (feats, codes, data)."""
    seed = _draw_seed()
    probs = feature_probs.float().reshape(1, -1)
    x, nnz, idx, val = synth_rows(feats.to(device), probs, dataset_size, 0, dataset_size, seed, False, 0.0,
                                  code_cap=n_ground_truth_components)
    return feats, _dense_codes(seed, 0, nnz, idx, val, None, n_ground_truth_components), x


def generate_correlated_dataset(n_ground_truth_components: int, dataset_size: int, corr_matrix: torch.Tensor,
                                feats: torch.Tensor, frac_nonzero: float, decay: torch.Tensor,
                                device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """random_dataset.py:191-245: one correlated Gaussian draw for all rows, the zero-row rule. (feats, codes, data)."""
    seed = _draw_seed()
    z = group_gaussians(seed, 0, 1, n_ground_truth_components, device)
    probs = component_probs(z, _cholesky(corr_matrix.to(device)), decay.to(device), frac_nonzero)
    x, nnz, idx, val = synth_rows(feats.to(device), probs, dataset_size, 0, dataset_size, seed, True, 0.0,
                                  code_cap=n_ground_truth_components)
    return feats, _dense_codes(seed, 0, nnz, idx, val, probs, n_ground_truth_components), x


# ----------------------------------------------------------------------------------------------------------------
# generators
# ----------------------------------------------------------------------------------------------------------------
class _RowSource:
    """What both generators share: per-group probabilities, one group per send, and a (group, row) counter. Send g of
    ``rows`` rows holds global rows ``row .. row + rows - 1``, all keyed by the generator's ``seed``."""

    _zero_row_rule = True

    def _init_counters(self):
        if getattr(self, "seed", None) is None:
            self.seed = _draw_seed()
        self._group, self._row = 0, 0

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("_chol_cache", None)          # re-derived from the covariance after loading
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        if "_group" not in state:               # a generator.pt written by the reference: start a fresh stream
            self.seed = None
            self._init_counters()

    def _rows(self, group0: int, n_groups: int, rows_per_group: int, row0: int, out: Optional[torch.Tensor] = None):
        """Rows of groups group0 .. group0 + n_groups - 1, rows_per_group each, the first at global row row0, in
        t_type (fp16 or fp32 from the kernel, other types converted from fp32)."""
        probs = self._group_probs(group0, n_groups)
        kdtype = self.t_type if self.t_type in (torch.float16, torch.float32) else torch.float32
        x, _, _, _ = synth_rows(self._feats(), probs, rows_per_group, row0, n_groups * rows_per_group, self.seed,
                                self._zero_row_rule, self._noise_scale(), kdtype, out=out)
        return x if x.dtype == self.t_type else x.to(self.t_type)

    def sends(self, n: int, batch_size: Optional[int] = None) -> torch.Tensor:
        """``n`` consecutive sends in one kernel call: [n * batch_size, d], equal to ``torch.cat`` of n ``send``s."""
        rows = self.batch_size if batch_size is None else int(batch_size)
        x = self._rows(self._group, n, rows, self._row)
        self._group += n
        self._row += n * rows
        return x

    def throw(self, type: Any = None, value: Any = None, traceback: Any = None) -> None:
        raise StopIteration


@dataclass
class SparseMixDataset(_RowSource, Generator):
    """random_dataset.py:76-142: sparse components with correlated activation probabilities plus Gaussian noise;
    the generator of big_sweep's synthetic sweep. ``seed``: the generator's random stream (None: one draw from torch's
    default generator). Rows are made by sce_synth_rows: ``activation_dim`` a multiple of 8 in [8, 8192]."""
    activation_dim: int
    n_sparse_components: int
    batch_size: int
    feature_num_nonzero: int
    feature_prob_decay: float
    noise_magnitude_scale: float
    device: Union[torch.device, str]

    sparse_component_dict: Optional[torch.Tensor] = None
    sparse_component_covariance: Optional[torch.Tensor] = None
    noise_covariance: Optional[torch.Tensor] = None
    t_type: Optional[torch.dtype] = None
    seed: Optional[int] = None

    sparse_component_probs: Optional[torch.Tensor] = field(init=False)

    def __post_init__(self):
        self.frac_nonzero = self.feature_num_nonzero / self.n_sparse_components
        if self.sparse_component_dict is None:
            self.sparse_component_dict = generate_rand_feats(self.activation_dim, self.n_sparse_components,
                                                             device=self.device)
        if self.sparse_component_covariance is None:
            self.sparse_component_covariance = generate_corr_matrix(self.n_sparse_components, device=self.device)
        if self.noise_covariance is None:
            self.noise_covariance = torch.eye(self.activation_dim, device=self.device)
        if not _is_identity(self.noise_covariance):
            raise NotImplementedError("only the identity noise covariance is generated (the one every caller uses)")
        self.sparse_component_probs = torch.tensor(
            [self.feature_prob_decay ** i for i in range(self.n_sparse_components)], dtype=torch.float32).to(self.device)
        if self.t_type is None:
            self.t_type = torch.float32
        self._init_counters()

    def _feats(self):
        return self.sparse_component_dict

    def _noise_scale(self):
        return self.noise_magnitude_scale

    def _group_probs(self, group0: int, n_groups: int) -> torch.Tensor:
        if "_chol_cache" not in self.__dict__:
            self._chol_cache = _cholesky(self.sparse_component_covariance)
        z = group_gaussians(self.seed, group0, n_groups, self.n_sparse_components, self.sparse_component_probs.device)
        return component_probs(z, self._chol_cache, self.sparse_component_probs, self.frac_nonzero)

    def send(self, batch_size: Optional[int] = None) -> torch.Tensor:
        return self.sends(1, batch_size)


@dataclass
class RandomDatasetGenerator(_RowSource, Generator):
    """random_dataset.py:16-73: fixed probabilities ``decay * frac_nonzero`` (no zero-row rule, no noise), or with
    ``correlated`` one correlated draw per send as SparseMixDataset without noise; fp32 rows."""
    activation_dim: int
    n_ground_truth_components: int
    batch_size: int
    feature_num_nonzero: int
    feature_prob_decay: float
    correlated: bool
    device: Union[torch.device, str]
    seed: Optional[int] = None

    frac_nonzero: float = field(init=False)
    decay: torch.Tensor = field(init=False)
    feats: torch.Tensor = field(init=False)
    corr_matrix: Optional[torch.Tensor] = field(init=False)
    component_probs: Optional[torch.Tensor] = field(init=False)

    def __post_init__(self):
        self.frac_nonzero = self.feature_num_nonzero / self.n_ground_truth_components
        self.decay = torch.tensor([self.feature_prob_decay ** i for i in range(self.n_ground_truth_components)]).to(
            self.device)
        self.corr_matrix = self.component_probs = None
        if self.correlated:
            self.corr_matrix = generate_corr_matrix(self.n_ground_truth_components, device=self.device)
        else:
            self.component_probs = self.decay * self.frac_nonzero
        self.feats = generate_rand_feats(self.activation_dim, self.n_ground_truth_components, device=self.device)
        self.t_type = torch.float32
        self._init_counters()

    @property
    def _zero_row_rule(self) -> bool:
        # generate_correlated_dataset fills empty rows, generate_rand_dataset does not; derived from the field so that
        # a pickle without it (the reference's) gets the rule of its own path
        return self.correlated

    def _feats(self):
        return self.feats

    def _noise_scale(self):
        return 0.0

    def _group_probs(self, group0: int, n_groups: int) -> torch.Tensor:
        if not self.correlated:
            return self.component_probs.float().reshape(1, -1).expand(n_groups, -1)
        if "_chol_cache" not in self.__dict__:
            self._chol_cache = _cholesky(self.corr_matrix)
        z = group_gaussians(self.seed, group0, n_groups, self.n_ground_truth_components, self.decay.device)
        return component_probs(z, self._chol_cache, self.decay, self.frac_nonzero)

    def send(self, ignored_arg: Any = None) -> torch.Tensor:
        return self.sends(1)


for _cls in (SparseMixDataset, RandomDatasetGenerator):
    _cls.__module__ = _REF_MODULE


# ----------------------------------------------------------------------------------------------------------------
# chunks: files (big_sweep.py:228-237, 269-295) and file-free
# ----------------------------------------------------------------------------------------------------------------
def chunk_rows_for(activation_width: int, chunk_size_gb) -> int:
    """big_sweep.py:288-289: the rows of a chunk of ``chunk_size_gb`` GiB of fp16 activations (2**21 at d = 512 and
    2 GB). The size is cast to int bytes first: the reference's float default (config.py:45) makes its torch.zeros raise."""
    return int(chunk_size_gb * 1024 ** 3) // (activation_width * 2)


def generate_synthetic_dataset(cfg, generator, chunk_size: int, n_chunks: int) -> None:
    """big_sweep.py:228-237: ``{i}.pt`` in ``cfg.dataset_folder`` for i < n_chunks, each an fp32 [chunk_size, d] tensor
    holding ``chunk_size // batch_size`` consecutive sends (in the generator's t_type, fp16 for big_sweep), the rows past
    the last full send zero. One kernel call and one device-to-host copy per chunk instead of one per send."""
    bs = generator.batch_size
    n_samples = chunk_size // bs
    for i in range(n_chunks):
        chunk = torch.zeros((chunk_size, cfg.activation_width), dtype=torch.float32, device="cpu")
        if n_samples:
            chunk[:n_samples * bs] = generator.sends(n_samples).cpu()
        torch.save(chunk, os.path.join(cfg.dataset_folder, f"{i}.pt"))


def init_synthetic_dataset(cfg):
    """big_sweep.py:269-295: when ``cfg.dataset_folder`` is empty, build big_sweep's SparseMixDataset (identity
    covariance unless ``cfg.correlated_components``, fp16 rows), write ``cfg.n_chunks`` chunks and pickle the generator
    to ``cfg.output_folder/generator.pt``. Returns the generator (None when the folder already held chunks)."""
    os.makedirs(cfg.dataset_folder, exist_ok=True)
    os.makedirs(cfg.output_folder, exist_ok=True)
    if len(os.listdir(cfg.dataset_folder)) != 0:
        return None
    device = getattr(cfg, "device", "cuda:0")
    generator = SparseMixDataset(
        cfg.activation_width, cfg.n_ground_truth_components, cfg.gen_batch_size, cfg.feature_num_nonzero,
        cfg.feature_prob_decay, cfg.noise_magnitude_scale, device,
        sparse_component_covariance=None if cfg.correlated_components
        else torch.eye(cfg.n_ground_truth_components, device=device),
        t_type=torch.float16)
    generate_synthetic_dataset(cfg, generator, chunk_rows_for(cfg.activation_width, cfg.chunk_size_gb), cfg.n_chunks)
    torch.save(generator, os.path.join(cfg.output_folder, "generator.pt"))
    return generator


class SyntheticChunks:
    """Device-resident chunks of ``generator`` for ``train_on_chunks(chunks=...)``: iterates ``(chunk_idx, chunk)``
    over ``order`` (default ``range(n_chunks)``) as ChunkStreamer does over files. Chunk i holds sends
    i S .. i S + S - 1 (S = chunk_rows // batch_size, global rows i S batch_size onwards, i.e. rows
    [i chunk_rows, (i + 1) chunk_rows) when batch_size divides chunk_rows), rows past the last full send zero: the rows
    ``generate_synthetic_dataset`` writes to ``{i}.pt`` from a fresh generator, in the generator's t_type. Each chunk
    is generated when it is reached, bitwise the same every time, on every GPU."""

    def __init__(self, generator, n_chunks: int, chunk_rows: int, order: Optional[Iterable[int]] = None):
        if chunk_rows < generator.batch_size:
            raise ValueError(f"chunk_rows ({chunk_rows}) must hold at least one send of {generator.batch_size} rows")
        self.generator, self.n_chunks, self.chunk_rows = generator, int(n_chunks), int(chunk_rows)
        self.order = list(range(self.n_chunks)) if order is None else [int(i) for i in order]
        if any(i < 0 or i >= self.n_chunks for i in self.order):
            raise ValueError(f"chunk indices must lie in [0, {self.n_chunks})")

    def __len__(self) -> int:
        return len(self.order)

    def chunk(self, i: int) -> torch.Tensor:
        g = self.generator
        sends = self.chunk_rows // g.batch_size
        rows = sends * g.batch_size
        dev = g._feats().device
        x = torch.zeros(self.chunk_rows, g.activation_dim, dtype=g.t_type, device=dev)
        if g.t_type in (torch.float16, torch.float32):
            g._rows(i * sends, sends, g.batch_size, i * rows, out=x[:rows])
        else:
            x[:rows] = g._rows(i * sends, sends, g.batch_size, i * rows)
        return x

    def __iter__(self):
        for i in self.order:
            yield i, self.chunk(i)
