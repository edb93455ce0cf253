"""ICA baseline (reference ``autoencoders/ica.py``): ``ICAEncoder``, sklearn's ``StandardScaler`` then ``FastICA()``
(parallel updates, logcosh, unit-variance whitening), fitted on the GPU. ``sweep_baselines.py`` saves it as ``ica.pt``
and its top-k export as ``ica_topk.pt``.

The fit, with m, s the column mean and population std of x, C its population covariance and N rows:
  * Whitening. The eigenpairs (lam, u) of the correlation D^-1 C D^-1 (D = diag(s)), in descending order with each u
    signed by its first entry, are the left singular vectors of the centred standardised rows, with sigma^2 = N lam.
    So FastICA's whitening_ is K = (u / sqrt(N lam))^T and the whitened rows are X1 = Kw (x - m)^T with
    Kw = diag(1 / sqrt(lam)) u^T D^-1. C and m come from one ``sce_second_moments`` pass (``BatchedPCA``).
  * Iterations. Each runs ``sce_ica_pass`` over the rows with unmix = W Kw folded into one fp32 matrix, so no whitened
    copy of the rows is ever written: G X1^T / N = gx Kw^T / N and mean_b g' = g_sum / N. The update, the symmetric
    decorrelation (``eigh`` of W W^T) and lim run in fp64 on the device; lim is the one value read back per
    iteration.
    The engine's shift is the fp32 column mean; it differs from m by less than the fp32 rounding v itself carries.
  * Unit variance. The sources' std is sqrt(diag(W W^T) / N) in exact arithmetic (K Sigma_z K^T = I / N), so no data
    pass is needed for it. components_ = W K, mixing_ = pinv(components_) in fp64.

The fitted state keeps sklearn's attribute names as numpy float64 arrays (``ica.ica.components_``, ``ica.scaler.mean_``),
in small project classes: sklearn is not needed to fit or to encode. ``encode`` reads only the attributes sklearn's
objects share, so an ``ica.pt`` the reference saved encodes through this class wherever sklearn can unpickle it.

Deliberate differences: fp64 input is fitted as fp32 rows (the engine reads fp16 or fp32); ``to_topk_dict`` passes
unit-norm torch rows (the reference passes raw numpy components_, which its own TopKLearnedDict.encode cannot take);
``to_nneg_dict`` is not mirrored (see there); rank-deficient data raises instead of dividing by ~0."""
from __future__ import annotations

import warnings

import numpy as np
import torch

from ._rowpass import RowPasses, check_width, convergence_warning, device_rows, fit_device
from .learned_dict import LearnedDict
from .pca import BatchedPCA
from .topk_encoder import TopKLearnedDict

_REF_MODULE = "autoencoders.ica"


class FittedScaler:
    """StandardScaler's fitted attributes: ``mean_``, ``var_``, ``scale_`` (float64 [d]) and ``n_samples_seen_``."""

    def __init__(self, mean, var, scale, n_samples):
        self.mean_, self.var_, self.scale_ = mean, var, scale
        self.n_samples_seen_ = np.int64(n_samples)


class FittedFastICA:
    """FastICA's fitted attributes: ``components_``, ``mixing_``, ``mean_``, ``whitening_``, ``_unmixing`` (float64)
    and ``n_iter_``."""

    def __init__(self, components, mixing, mean, whitening, unmixing, n_iter):
        self.components_, self.mixing_, self.mean_ = components, mixing, mean
        self.whitening_, self._unmixing, self.n_iter_ = whitening, unmixing, int(n_iter)


def _sym_decorrelation(W):
    s, u = torch.linalg.eigh(W @ W.T)
    s = s.clamp(min=torch.finfo(W.dtype).tiny)
    return (u * s.rsqrt()) @ u.T @ W


class ICAEncoder(LearnedDict):
    """ica.py:18-58. ``activation_size``: d (a multiple of 8 to fit; 16 for ``arith="f16f8"``). ``n_components`` sets
    ``n_feats`` only, as in the reference, whose FastICA() always fits d components. ``device``: the CUDA device of
    the fit (default: the current one). ``max_iter``, ``tol``, ``alpha`` and ``w_init`` carry FastICA's names and
    defaults; ``w_init=None`` draws ``np.random.normal(size=(d, d))`` from numpy's global RNG at ``train``, as sklearn
    does, so ``np.random.seed`` reproduces the reference's fit."""

    def __init__(self, activation_size, n_components: int = 0, *, device=None, arith: str = "auto", max_iter=200,
                 tol=1e-4, alpha=1.0, w_init=None):
        self.activation_size = activation_size
        self.n_feats = n_components if n_components else activation_size
        self.device = device
        self.arith = arith
        self.max_iter, self.tol, self.alpha, self.w_init = int(max_iter), float(tol), float(alpha), w_init
        self.ica = None
        self.scaler = None

    def to_device(self, device):
        pass

    # ---- fitting
    def _device(self):
        return fit_device(self.device if self.device is not None else "cuda")

    def fit(self, dataset):
        """Fits the scaler and FastICA to the rows of ``dataset`` [N, d] and returns ``self``; ``train`` also returns the
        sources."""
        d = int(self.activation_size)
        check_width(d, self.arith)
        if not 1.0 <= self.alpha <= 2.0:
            raise ValueError(f"alpha must be in [1, 2], got {self.alpha}")
        x = torch.as_tensor(dataset)
        if x.dim() != 2 or x.shape[1] != d:
            raise ValueError(f"dataset must be [N, {d}], got {tuple(x.shape)}")
        if x.shape[0] < 2:
            raise ValueError("ICA needs at least two rows")
        dev = self._device()
        x = device_rows(x, dev)
        N = x.shape[0]
        w_init = np.random.normal(size=(d, d)) if self.w_init is None else np.asarray(self.w_init, dtype=np.float64)
        if w_init.shape != (d, d):
            raise ValueError(f"w_init must be [{d}, {d}], got {w_init.shape}")
        # ---- standardise and whiten from one second-moment pass
        pca = BatchedPCA(d, dev, arith=self.arith)
        pca.train_batch(x)
        pca._ready()
        m, cov = pca._mean64(), pca._cov64()
        cov = 0.5 * (cov + cov.T)
        if not bool(torch.isfinite(cov).all()):
            raise ValueError("the rows hold a non-finite value: their covariance is not finite")
        var = cov.diagonal().clone()
        eps = torch.finfo(torch.float64).eps
        scale = torch.where(var <= N * eps * var + (N * m * eps) ** 2, torch.ones_like(var), var.clamp(min=0).sqrt())
        corr = cov / torch.outer(scale, scale)
        lam, u = torch.linalg.eigh(0.5 * (corr + corr.T))
        lam, u = lam.flip(0), u.flip(1)
        if not bool(lam[-1] > d * eps * lam[0]):
            raise ValueError(f"the standardised data are rank-deficient (correlation eigenvalues {float(lam[0]):.3e} .. "
                             f"{float(lam[-1]):.3e}): FastICA's whitening is undefined")
        u = u * torch.sign(u[0])
        K = (u / (N * lam).sqrt()).T
        Kw = (u / lam.sqrt()).T / scale
        # ---- iterations
        passes = RowPasses(d, dev, self.arith)
        g_sum = torch.empty(d, dtype=torch.float64, device=dev)
        gx = torch.empty(d, d, dtype=torch.float64, device=dev)
        W = _sym_decorrelation(torch.as_tensor(w_init, dtype=torch.float64).to(dev))
        n_iter, lim = 0, float("inf")
        with torch.cuda.device(dev):
            for n_iter in range(1, self.max_iter + 1):
                unmix = (W @ Kw).float().contiguous()
                g_sum.zero_()
                gx.zero_()
                passes.ica_pass(x, pca.shift, unmix, self.alpha, g_sum, gx)
                W1 = _sym_decorrelation(gx @ Kw.T / N - (g_sum / N)[:, None] * W)
                lim_t = ((W1 * W).sum(dim=1).abs() - 1).abs().max()
                W = W1
                lim = float(lim_t)
                if lim < self.tol:
                    break
        passes.check_flag("the rows or the unmixing matrix")
        if not lim < self.tol:
            warnings.warn("FastICA did not converge. Consider increasing tolerance or the maximum number of "
                          "iterations.", convergence_warning())
        # ---- unit variance and the read-out
        W = W / ((W * W).sum(dim=1, keepdim=True) / N).sqrt()
        comp = W @ K
        np64 = lambda t: t.cpu().numpy().astype(np.float64)
        self.scaler = FittedScaler(np64(m), np64(var), np64(scale), N)
        self.ica = FittedFastICA(np64(comp), np64(torch.linalg.pinv(comp)), np.zeros(d), np64(K), np64(W), n_iter)
        return self

    def train(self, dataset):
        """Fits, then returns the sources of the rows, float64 [N, d] on ``dataset``'s device: N d 8 bytes (34 GB for
        2^21 rows of width 2048), computed in blocks on the fit's device."""
        self.fit(dataset)
        x = torch.as_tensor(dataset)
        out = torch.empty(x.shape, dtype=torch.float64, device=x.device)
        dev = self._device()
        step = max(1, (1 << 27) // max(1, x.shape[1]))
        for s in range(0, x.shape[0], step):
            out[s:s + step] = self._encode64(x[s:s + step].to(dev)).to(x.device)
        return out

    # ---- read-out
    def _encode64(self, x):
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64), device=x.device)
        z = (x.double() - t(self.scaler.mean_)) / t(self.scaler.scale_)
        return (z - t(self.ica.mean_)) @ t(self.ica.components_).T

    def encode(self, x):
        """((x - scaler.mean_) / scaler.scale_ - ica.mean_) @ ica.components_^T in float64, on ``x.device``."""
        assert x.shape[1] == self.activation_size
        return self._encode64(x)

    def get_learned_dict(self):
        """The components with unit-norm rows, fp32 (CPU), as in the reference."""
        comps = torch.tensor(self.ica.components_, dtype=torch.float32)
        return comps / torch.norm(comps, dim=-1, keepdim=True)

    def to_topk_dict(self, sparsity):
        """A TopKLearnedDict of the components and their negatives with unit-norm rows, fp32 torch. The reference passes
        the raw numpy components_, which its TopKLearnedDict.encode cannot multiply; evaluate_dicts' top-k plan
        normalises rows anyway, so with unit rows this export's own encode and evaluate_dicts agree."""
        rows = self.get_learned_dict()
        return TopKLearnedDict(torch.cat((rows, -rows)), sparsity)

    def to_nneg_dict(self):
        raise NotImplementedError(
            "NNegICAEncoder is not mirrored: the reference's encode reads a self.scaler it never sets and calls "
            "np.clamp, which does not exist, so it cannot run")


for _cls in (ICAEncoder, FittedScaler, FittedFastICA):
    _cls.__module__ = _REF_MODULE
