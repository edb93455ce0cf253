"""NMF baseline (reference ``autoencoders/nmf.py``): ``NMFEncoder``, sklearn's ``NMF()`` with its defaults (coordinate
descent, Frobenius loss, NNDSVDA start, tol 1e-4, at most 200 iterations, no regularisation, coordinates in order),
fitted and applied on the GPU. It always fits k = d components, as the reference's ``NMF()`` does.

The fit, for the rows v = x - shift (>= 0 after the shift rule) of an [N, d] dataset:
  * NNDSVDA start. One ``sce_second_moments`` pass (with the shift as its shift vector) gives V^T V and the column sums;
    ``eigh`` of V^T V in fp64 gives the right singular vectors and S^2. Eigenvalues at or below d eps lambda_0 count as
    zero singular values, whose components NNDSVDA fills with the average. One ``sce_nmf_project`` pass with M = the
    singular vectors writes P = V M^T (= U S) into the resident W and the squared norms of the positive and negative
    parts of its columns; W_0 and H_0 then follow on the device from P, those norms and the eps / average rules.
  * Iterations. Per row block: ``sce_nmf_project`` with M = H gives X H^T, then the fp32 ``sce_nmf_cd_sweep`` updates
    that block of W with G = H H^T; ``sce_nmf_grams`` then adds the block's W^T W and W^T X. The fp64 sweep updates
    H^T with W^T W and X^T W. The violation of both sweeps is one fp64 scalar on the device, read back once per
    iteration for sklearn's stop rule.
  * reconstruction_err_ = ||X - W H||_F from one ``sce_nmf_residual`` pass, fp32 products on the CUDA cores with the
    squares in fp64. The expansion ||X||^2 - 2 <W^T X, H> + <W^T W, H H^T> would need no extra pass, but it cancels
    the digits that matter: at fits whose error is 6e-3 and 6e-4 of ||X|| (rank12 and sep16 of the tests), bf16x3
    Grams (each product good to ~2^-16) left it 7 % off and at zero.
W stays resident in fp32: N d 4 bytes, 4 GiB at d = 512 and 16 GiB at d = 2048 for 2^21 rows.

Accuracy. The projections and Grams run in bf16x3, whose products are good to ~2^-16, not fp32's 2^-24 (an fp32
operand is carried as two bf16 planes and lo*lo is dropped). On well-conditioned data the fit and transform land within
1e-4 of sklearn's fp64 ones. On ill-conditioned data they do not: where H H^T has a condition number near 1e6, transform's
codes land up to ~1.2e-3 from sklearn's (with X H^T in fp32 they would land within 3e-5), and a fit whose NNDSVDA start
comes from a Gram matrix with eigenvalues spanning 6 orders of magnitude ends up to ~3e-2 away after 200 iterations.
The iteration and sweep counts match sklearn's.

``encode`` is sklearn's ``transform``: the W-update alone from W = 0 with H fixed, up to max_iter sweeps with the same
stop rule over the whole batch (so a row's code depends on the batch it came in). The sweeps queue on the device with
their stop state there (``sce_nmf_cd_sweep``'s n_iter form), so no sweep waits for the host.

The fitted state keeps sklearn's attribute names (``enc.nmf.components_`` float64, ``n_iter_``, ...) in a small project
class: sklearn is not needed to fit or to encode. ``encode`` reads only ``components_``, ``max_iter`` and ``tol``, which
sklearn's ``NMF`` shares, so an ``nmf.pt`` the reference saved encodes through this class wherever sklearn can unpickle
it.

Deliberate differences: the caller's tensors are never modified (the reference subtracts the shift from them in place in
``train`` and ``encode``, and clamps in ``encode``); fp32 datasets are fitted too, and still encode (the reference fits
them in fp32 and its ``encode`` then raises a TypeError); N < d raises (sklearn would switch to a random start); fp64
input is fitted as fp32 rows (the engine reads fp16 or fp32)."""
from __future__ import annotations

import ctypes as C
import warnings

import numpy as np
import torch

from . import _lib
from ._rowpass import RowPasses, call_rows, check_width, convergence_warning, device_rows, fit_device
from .learned_dict import LearnedDict
from .topk_encoder import TopKLearnedDict

_REF_MODULE = "autoencoders.nmf"
_EPS_INIT = 1e-6      # sklearn's _initialize_nmf eps
_MAX_K = 2048         # sce_nmf_cd_sweep's widest row
_FLAG_WHAT = "the rows or the factors"


class FittedNMF:
    """sklearn NMF's fitted attributes: ``components_`` (float64 [k, d]), ``n_components_``, ``n_iter_``,
    ``reconstruction_err_``, ``n_features_in_``, and the ``tol`` / ``max_iter`` that ``transform`` uses."""

    def __init__(self, components, n_iter, reconstruction_err, tol, max_iter):
        self.components_ = components
        self.n_components_, self.n_features_in_ = components.shape
        self.n_iter_ = int(n_iter)
        self.reconstruction_err_ = float(reconstruction_err)
        self.tol, self.max_iter = float(tol), int(max_iter)


def _gram(H):
    """H H^T, exactly symmetric: sce_nmf_cd_sweep reads G[t][:] for G's column t as well."""
    G = H @ H.T
    return 0.5 * (G + G.T)


def _cd_sweep(w, w_is_f64, k, g, l, ws, viol, max_sweeps=1, tol=0.0, n_iter=None):
    """sce_nmf_cd_sweep over the rows of w [R, k] on the current stream; ``ws``: (tensor, address) of its workspace."""
    lib, stream = _lib.load(), C.c_void_p(torch.cuda.current_stream(w.device).cuda_stream)
    _lib.check(lib.sce_nmf_cd_sweep(w.data_ptr(), w_is_f64, w.shape[0], k, g.data_ptr(), l.data_ptr(), max_sweeps,
                                    C.c_double(tol), viol.data_ptr(), None if n_iter is None else n_iter.data_ptr(),
                                    ws[1], ws[0].numel() - 1024, stream), "sce_nmf_cd_sweep")


class NMFEncoder(LearnedDict):
    """nmf.py:29-67. ``activation_size``: d, a multiple of 8 up to 2048 (16 for ``arith="f16f8"``). ``n_components``
    sets ``n_feats`` only, as in the reference, whose NMF() always fits d components. ``shift``: subtracted from the
    rows; ``train`` lowers it to the dataset's minimum when that is below it, as the reference does. ``device``: the
    CUDA device of the fit and of ``encode`` (default: the current one). ``max_iter`` and ``tol`` carry NMF's names
    and defaults."""

    def __init__(self, activation_size, n_components: int = 0, shift=0.0, *, device=None, arith: str = "auto",
                 max_iter=200, tol=1e-4):
        self.activation_size = activation_size
        self.n_feats = n_components if n_components else activation_size
        self.nmf = None
        self.shift = shift
        self.device = device
        self.arith = arith
        self.max_iter, self.tol = int(max_iter), float(tol)

    def to_device(self, device):
        pass

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("_cache", None)
        return state

    # ---- helpers
    def _device(self, fallback=None):
        dev = getattr(self, "device", None)
        if dev is None:
            dev = fallback if fallback is not None and torch.device(fallback).type == "cuda" else "cuda"
        return fit_device(dev)

    # ---- fitting
    def fit(self, dataset):
        """Fits NMF to the rows of ``dataset`` [N, d] (after the shift rule) and returns ``self``."""
        self.fit_transform(dataset)
        return self

    def fit_transform(self, dataset):
        """Fits as ``fit`` and returns the fitted codes W, fp32 [N, d] on the fit device (sklearn's fit_transform)."""
        return self._fit(dataset)[0]

    def _fit(self, dataset):
        """(W, the violation of each iteration): the fit behind ``fit`` and ``fit_transform``."""
        d = int(self.activation_size)
        arith = getattr(self, "arith", "auto")
        check_width(d, arith, _MAX_K)
        x_in = torch.as_tensor(dataset)
        if x_in.dim() != 2 or x_in.shape[1] != d:
            raise ValueError(f"dataset must be [N, {d}], got {tuple(x_in.shape)}")
        N = x_in.shape[0]
        if N < d:
            raise ValueError(f"NNDSVDA needs at least d = {d} rows, got {N} (sklearn would start from random factors)")
        # the shift rule of nmf.py:51-52: the caller's tensor is not modified
        lo = torch.min(x_in)
        if lo < self.shift:
            self.shift = lo
        dev = self._device(x_in.device)
        x = device_rows(x_in, dev)
        passes = RowPasses(d, dev, arith)
        B0 = min(call_rows(d), N)
        cd_ws = _lib.workspace(max(_lib.load().sce_nmf_cd_sweep_workspace_bytes(d, R) for R in (B0, d)), dev,
                               "sce_nmf_cd_sweep_workspace_bytes")
        f64 = dict(dtype=torch.float64, device=dev)
        shift_vec = torch.full((d,), float(self.shift), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            # ---- NNDSVDA
            col_sum, gram = torch.zeros(d, **f64), torch.zeros(d, d, **f64)
            passes.second_moments(x, shift_vec, col_sum, gram)
            passes.check_flag(_FLAG_WHAT)
            if not bool(torch.isfinite(gram).all()):
                raise ValueError("the rows hold a non-finite value")
            avg = float(col_sum.sum()) / (N * d)
            lam, vec = torch.linalg.eigh(0.5 * (gram + gram.T))
            lam, vec = lam.flip(0), vec.flip(1)
            if not float(lam[0]) > 0:
                raise ValueError("the shifted rows are all zero: NMF has nothing to fit")
            zero = lam <= d * torch.finfo(torch.float64).eps * lam[0]
            S = torch.where(zero, torch.zeros_like(lam), lam.clamp(min=0).sqrt())
            Vr = vec.T.contiguous()                      # rows: the right singular vectors
            W = torch.empty(N, d, dtype=torch.float32, device=dev)
            norms = torch.zeros(2 * d, **f64)
            passes.nmf_project(x, shift_vec, Vr.float().contiguous(), W, norms)
            pos, neg = norms[:d], norms[d:]
            yp, yn = Vr.clamp(min=0), (-Vr).clamp(min=0)
            ypn, ynn = yp.norm(dim=1), yn.norm(dim=1)
            Ssafe = torch.where(zero, torch.ones_like(S), S)
            mp, mn = pos.sqrt() / Ssafe * ypn, neg.sqrt() / Ssafe * ynn
            use_p = mp > mn
            lbd = (S * torch.where(use_p, mp, mn)).sqrt()
            w_scale = lbd / torch.where(use_p, pos, neg).sqrt()
            w_sign = torch.where(use_p, 1.0, -1.0).to(torch.float64)
            H = lbd[:, None] * torch.where(use_p[:, None], yp / ypn[:, None], yn / ynn[:, None])
            # the leading pair is non-negative up to its sign: sklearn takes the absolute values
            w_scale[0], w_sign[0] = 1.0 / S[0].sqrt(), 1.0
            H[0] = S[0].sqrt() * Vr[0].abs()
            w_scale = torch.nan_to_num(torch.where(zero, 0.0, w_scale), nan=0.0, posinf=0.0).float()
            w_sign = w_sign.float()
            H = torch.nan_to_num(torch.where(zero[:, None], 0.0, H), nan=0.0)
            for blk in W.split(call_rows(d)):
                blk[:, 0].abs_()
                blk.mul_(w_sign).clamp_(min=0).mul_(w_scale)
                blk.masked_fill_(blk < _EPS_INIT, avg)
            H = torch.where(H < _EPS_INIT, torch.full_like(H, avg), H)
            # ---- iterations
            L = torch.empty(B0, d, dtype=torch.float32, device=dev)
            wtw, wtv = torch.zeros(d, d, **f64), torch.zeros(d, d, **f64)
            viol = torch.zeros(1, **f64)
            v0, n_iter, violations = None, 0, []
            for n_iter in range(1, self.max_iter + 1):
                Hf = H.float().contiguous()
                G = _gram(H).float().contiguous()
                viol.zero_()
                wtw.zero_()
                wtv.zero_()
                for xb, wb in zip(x.split(B0), W.split(B0)):
                    passes.nmf_project(xb, shift_vec, Hf, L)
                    _cd_sweep(wb, 0, d, G, L, cd_ws, viol)
                    passes.nmf_grams(xb, shift_vec, wb, wtw, wtv)
                Ht = H.T.contiguous()
                Lh = wtv.T.contiguous()
                wtw_s = (0.5 * (wtw + wtw.T)).contiguous()   # the sweep reads G[t][:] as its column t too
                _cd_sweep(Ht, 1, d, wtw_s, Lh, cd_ws, viol)
                H = Ht.T.contiguous()
                v = float(viol)
                violations.append(v)
                if n_iter == 1:
                    v0 = v
                if v0 == 0 or v / v0 <= self.tol:
                    break
            # ---- reconstruction_err_: one fp32 residual pass over the rows
            Hf = H.float().contiguous()
            res = torch.zeros(1, **f64)
            passes.nmf_residual(x, shift_vec, W, Hf, res)
        passes.check_flag(_FLAG_WHAT)
        if n_iter == self.max_iter and self.tol > 0:
            warnings.warn(f"Maximum number of iterations {self.max_iter} reached. Increase it to improve convergence.",
                          convergence_warning())
        self.nmf = FittedNMF(H.cpu().numpy().astype(np.float64), n_iter, float(res.sqrt()), self.tol, self.max_iter)
        self._cache = None
        return W, violations

    def train(self, dataset):
        """nmf.py:50-59: fits, returns None. Unlike the reference, ``dataset`` is left as it is."""
        self.fit(dataset)

    # ---- read-out
    def _factors(self, dev):
        """(H fp32 [k, d], H H^T fp32 [k, k]) on ``dev``, cached per device and components_."""
        comps = self.nmf.components_
        cache = getattr(self, "_cache", None)
        if cache is None or cache[0] != dev or cache[1] is not comps:
            H = torch.as_tensor(np.asarray(comps, dtype=np.float64), device=dev)
            cache = (dev, comps, H.float().contiguous(), _gram(H).float().contiguous())
            self._cache = cache
        return cache[2], cache[3]

    def transform(self, x):
        """(codes fp32 [B, k] on the fit device, the number of sweeps run): sklearn's NMF.transform of
        max(x - shift, 0)."""
        k, d = self.nmf.components_.shape
        if x.dim() != 2 or x.shape[1] != d:
            raise ValueError(f"x must be [B, {d}], got {tuple(x.shape)}")
        if k % 8 or k > _MAX_K:
            raise ValueError(f"the engine encodes k in multiples of 8 up to {_MAX_K} components, got {k}")
        dev = self._device(x.device)
        xs = device_rows(x, dev)
        B = xs.shape[0]
        passes = RowPasses(d, dev, getattr(self, "arith", "auto"))
        cd_ws = _lib.workspace(_lib.load().sce_nmf_cd_sweep_workspace_bytes(k, B), dev,
                               "sce_nmf_cd_sweep_workspace_bytes")
        with torch.cuda.device(dev):
            Hf, G = self._factors(dev)
            shift_vec = torch.full((d,), float(self.shift), dtype=torch.float32, device=dev)
            P = torch.empty(B, k, dtype=torch.float32, device=dev)
            passes.nmf_project(xs, shift_vec, Hf, P)
            W = torch.zeros(B, k, dtype=torch.float32, device=dev)
            viol = torch.empty(2, dtype=torch.float64, device=dev)
            n_it = torch.empty(1, dtype=torch.int32, device=dev)
            _cd_sweep(W, 0, k, G, P, cd_ws, viol, int(self.nmf.max_iter), float(self.nmf.tol), n_it)
        passes.check_flag(_FLAG_WHAT)
        return W, int(n_it.item())

    def encode(self, x):
        """nmf.py:43-49: the codes of max(x - shift, 0) from sklearn's transform, float64 on ``x.device``. ``x`` is not
        modified."""
        return self.transform(x)[0].double().to(x.device)

    def get_learned_dict(self):
        """The raw components, fp32 (CPU), as in the reference."""
        return torch.tensor(self.nmf.components_, dtype=torch.float32)

    def to_topk_dict(self, sparsity):
        """The reference's TopKLearnedDict of the raw components (rows not normalised), so that its own encode matches
        the reference's. ``metrics.evaluate_dicts`` normalises the rows of top-k dictionaries, so it would score a
        different dictionary than this export's encode uses."""
        return TopKLearnedDict(self.get_learned_dict(), sparsity)


for _cls in (NMFEncoder, FittedNMF):
    _cls.__module__ = _REF_MODULE
