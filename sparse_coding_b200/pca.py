"""PCA baselines (reference ``autoencoders/pca.py``): the streaming covariance of a set of activations, fitted on the
GPU, and the dictionaries the sweeps and plots compare against (``sweep_baselines.py:56-73``, the "PCA (TopK)" and
"PCA (Static)" curves of ``plotting/fvu_sparsity_plot*.py:143-161``).

The reference's ``train_batch`` forms a ``[B, d, d]`` outer-product tensor per batch. Here the fit is one Gram matrix per
engine call (libsce ``sce_second_moments``): the rows, shifted by a fixed vector, are split into operand planes and
multiplied on the split-operand GEMM, and their column sums and Gram matrix accumulate in fp64 on the device.

Read-out. With the shift s, N rows x_b and v_b = x_b - s, the object holds S1 = sum_b v_b and S2 = sum_b v_b v_b^T:

    mean = s + S1 / N
    cov  = (S2 - S1 S1^T / N) / N = (1/N) sum_b (x_b - mean)(x_b - mean)^T        (population covariance)

The reference's batch merge (pca.py:57-63) computes the same quantity in exact arithmetic. With the running mean m_a and
covariance C_a of n_a rows, a batch of n_b rows, delta = mean_b - m_a and n = n_a + n_b, it sets
    m = m_a + delta n_b / n,
    C = C_a n_a / n + (1/n) sum_b (x_b - m_a)(x_b - m)^T.
Writing x_b - m_a = (x_b - mean_b) + delta and x_b - m = (x_b - mean_b) + delta n_a / n, the sum is
n_b C_b + n_b delta delta^T n_a / n (the cross terms vanish), so C n = n_a C_a + n_b C_b + delta delta^T n_a n_b / n:
Chan et al.'s pairwise update of the sum of squared deviations, which by induction equals sum (x - mean)(x - mean)^T
over all rows. That is S2 - S1 S1^T / N for any fixed s.

The shift is the first batch's column mean (computed in fp64, stored in fp32), so that v is small against the offset of
typical activations and the subtraction S1 S1^T / N cancels little. The first row would be a poor shift: the first row
of a language-model chunk is often a BOS outlier.

Reference quirks kept, so that the exports stay drop-ins:
  * ``get_centering_transform`` returns the eigenvectors in COLUMNS while ``TiedSAE.center`` multiplies by
    ``rot.T``: fed to ``FunctionalTiedSAE.init(translation=, rotation=, scaling=)`` it does not project onto the
    eigenbasis. Reproduced as it is.
  * ``to_rotation_dict`` returns a ``Rotation`` on the CPU (its ``device=None`` default).
  * Eigenvector signs are whatever ``torch.linalg.eigh`` gives.
Deliberate difference: ``to_pve_rotation_dict`` puts the zero bias on the dictionary's device; the reference creates it
on the CPU beside device rows.

``BatchedMean`` / ``calc_mean`` are not mirrored: no caller uses them (SURVEY, quirks)."""
from __future__ import annotations

import torch

from ._rowpass import RowPasses, check_width, cuts, fit_device
from .learned_dict import LearnedDict, Rotation, TiedSAE
from .topk_encoder import TopKLearnedDict

_REF_MODULE = "autoencoders.pca"


class BatchedPCA:
    """pca.py:41-110. ``n_dims``: activation width (a multiple of 8; 16 for ``arith="f16f8"``); ``device``: a CUDA
    device. ``arith``: the engine's operand arithmetic ("auto" runs bf16x3, which holds the fp32 range)."""

    def __init__(self, n_dims, device, arith: str = "auto"):
        self.n_dims = int(n_dims)
        self.device = fit_device(device)
        self.arith = arith
        check_width(self.n_dims, arith)
        d = self.n_dims
        self.n_samples = 0
        self.shift = None
        self.col_sum = torch.zeros(d, dtype=torch.float64, device=self.device)
        self.gram = torch.zeros(d, d, dtype=torch.float64, device=self.device)
        self._passes = RowPasses(d, self.device, arith)
        self._eig = None

    # ---- fitting
    def _check(self, activations):
        if not torch.is_tensor(activations) or activations.dim() != 2 or activations.shape[1] != self.n_dims:
            raise ValueError(f"activations must be a [B, {self.n_dims}] tensor, got "
                             f"{tuple(activations.shape) if torch.is_tensor(activations) else type(activations).__name__}")
        if activations.dtype not in (torch.float16, torch.float32):
            raise ValueError(f"activations must be fp16 or fp32, got {activations.dtype}")

    def _batches(self, activations, cuts):
        """The row ranges ``cuts`` of ``activations`` on the device, contiguous, in their own dtype."""
        if activations.device.type == "cuda":
            for s, e in cuts:
                yield activations[s:e].to(self.device).contiguous()
            return
        from .train_loop import HostBatchPrefetcher
        yield from HostBatchPrefetcher((activations[s:e].contiguous() for s, e in cuts), self.device)

    def train_batch(self, activations):
        """Adds the rows of ``activations`` [B, d] (fp16 or fp32, on a CUDA device or the CPU, B >= 1).

        The first batch also sets the shift (its column mean). When it takes one engine call (at most
        min(65536, 2^27 / d) rows: the reference's callers use 500 and 5000) the rows that call reads give the mean;
        a longer first batch is read once more for its mean first, so host input of that size crosses to the device
        twice."""
        self._check(activations)
        B = activations.shape[0]
        if B == 0:
            return
        calls = cuts(B, self.n_dims)
        col_sum = lambda xb: xb.sum(dim=0, dtype=torch.float64)
        with torch.cuda.device(self.device):
            if self.shift is None and len(calls) > 1:
                total = sum(col_sum(xb) for xb in self._batches(activations, calls))
                self.shift = (total / B).float().contiguous()
            for xb in self._batches(activations, calls):
                if self.shift is None:
                    self.shift = (col_sum(xb) / B).float().contiguous()
                self._passes.second_moments(xb, self.shift, self.col_sum, self.gram)
        self.n_samples += B
        self._eig = None

    # ---- read-out
    def _ready(self):
        if self.n_samples == 0:
            raise ValueError("BatchedPCA has seen no rows")
        self._passes.check_flag("the activations")

    def _mean64(self):
        return self.shift.double() + self.col_sum / self.n_samples

    def _cov64(self):
        n = self.n_samples
        return (self.gram - torch.outer(self.col_sum, self.col_sum) / n) / n

    def _decomposition(self):
        """The cached (eigenvalues ascending, eigenvectors in columns, fp32), shared by the exports: never handed out."""
        self._ready()
        if self._eig is None:
            cov = self._cov64()
            vals, vecs = torch.linalg.eigh(0.5 * (cov + cov.T))
            self._eig = (vals.float(), vecs.float())
        return self._eig

    def _directions(self, count=None):
        """The first ``count`` (default all) eigenvectors as rows, by eigenvalue, largest first."""
        vals, vecs = self._decomposition()
        order = vals.argsort(descending=True)
        return vecs.T[order[:count]]

    def get_mean(self):
        self._ready()
        return self._mean64().float()

    def get_pca(self):
        """(eigenvalues ascending [d], eigenvectors in columns [d, d]), fp32, of the symmetrised covariance; ``eigh`` runs
        in fp64 on the device once per fit state. Each call returns tensors of its own."""
        vals, vecs = self._decomposition()
        return vals.clone(), vecs.clone()

    def get_centering_transform(self):
        """(translation, rotation, scaling) = (mean, eigenvectors in columns, 1 / sqrt(max(eigenvalue, 1e-6)))."""
        vals, rot = self.get_pca()
        scaling = vals.clamp(min=1e-6).rsqrt()
        if bool(scaling.isnan().any()):
            raise ValueError("the covariance has a NaN eigenvalue: the centring scale is undefined")
        return self.get_mean(), rot, scaling

    def get_dict(self):
        return self._directions()

    def to_learned_dict(self, sparsity):
        return PCAEncoder(self._directions(), sparsity)

    def to_topk_dict(self, sparsity):
        rows = self._directions()
        return TopKLearnedDict(torch.cat((rows, -rows)), sparsity)

    def to_rotation_dict(self, n_components=None):
        return Rotation(self._directions(n_components))

    def to_pve_rotation_dict(self, n_components=None):
        """A centred TiedSAE of the first ``n_components`` directions and their negatives; its zero bias lies on the
        dictionary's device (the reference leaves it on the CPU)."""
        rows = self._directions(n_components)
        signed = torch.cat((rows, -rows))
        bias = signed.new_zeros(signed.shape[0])
        return TiedSAE(signed, bias, centering=(self.get_mean(), None, None), norm_encoder=True)


def calc_pca(activations, batch_size=512, device="cuda:0", arith: str = "auto"):
    """pca.py:6-13: a BatchedPCA of the whole of ``activations`` [N, d]. ``batch_size`` is accepted for the reference's
    signature; the engine's own rows per call decide the launches, and the result depends on it only through fp64
    rounding (the shift is the column mean of all N rows)."""
    pca = BatchedPCA(activations.shape[1], device, arith=arith)
    pca.train_batch(activations)
    return pca


class PCAEncoder(LearnedDict):
    """pca.py:113-135. ``pca_dict``: the directions, divided by their norms (no floor); ``sparsity``: k. The code keeps,
    per row, the k scores of largest magnitude with their signs and zeros elsewhere."""

    def __init__(self, pca_dict, sparsity):
        self.pca_dict = pca_dict / pca_dict.norm(dim=-1, keepdim=True)
        self.sparsity = sparsity
        self.n_feats, self.activation_size = self.pca_dict.shape

    def get_learned_dict(self):
        return self.pca_dict

    def to_device(self, device):
        self.pca_dict = self.pca_dict.to(device)

    def encode(self, batch):
        scores = batch @ self.pca_dict.T
        keep = scores.abs().topk(self.sparsity, dim=-1).indices
        return torch.zeros_like(scores).scatter(-1, keep, scores.gather(-1, keep))


PCAEncoder.__module__ = _REF_MODULE
