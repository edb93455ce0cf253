"""The row passes of libsce as the baselines use them (``sce_second_moments`` for BatchedPCA, ``sce_ica_pass`` for
ICAEncoder, ``sce_nmf_project`` / ``sce_nmf_grams`` / ``sce_nmf_residual`` for NMFEncoder): the fit device, the rows
per engine call, the rows on the device, and a ``RowPasses`` that holds what every call over rows of one width shares
(the arithmetic, the f16f8 range flag, one workspace) and loops each pass over the calls."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

_MAX_PLANE_ELEMS = 1 << 27       # rows per engine call x d: the planes of one call stay under ~0.8 GB
_MAX_CALL_ROWS = 1 << 16


def call_rows(d: int) -> int:
    """Rows per engine call at width d."""
    return max(64, min(_MAX_CALL_ROWS, _MAX_PLANE_ELEMS // d))


def cuts(N: int, d: int):
    """The (start, end) row ranges of the engine calls over N rows of width d."""
    step = call_rows(d)
    return [(s, min(s + step, N)) for s in range(0, N, step)]


def fit_device(device) -> torch.device:
    """``device`` as an indexed CUDA device; the engine has no CPU path."""
    dev = torch.device(device)
    if dev.type != "cuda" or not torch.cuda.is_available():
        raise RuntimeError(f"BatchedPCA fits in the sm_90a CUDA engine and needs a CUDA device (got {device!r}, CUDA "
                           f"available: {torch.cuda.is_available()}); there is no CPU implementation in the product path")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def convergence_warning():
    """The warning category sklearn would use; a UserWarning where sklearn is not installed. sklearn is imported only
    when a fit warns: importing it takes seconds, and BatchedPCA never needs it."""
    try:
        from sklearn.exceptions import ConvergenceWarning
    except ImportError:
        return UserWarning
    return ConvergenceWarning


def check_width(d: int, arith: str, max_d: int = 8192):
    if d < 8 or d % 8 or d > max_d or (_lib.arith_code(arith) == _lib.SCE_ARITH_F16F8 and d % 16):
        raise ValueError(f"the engine fits d in multiples of 8 (a multiple of 16 for f16f8) up to {max_d}, got {d}")


def device_rows(x, dev: torch.device) -> torch.Tensor:
    """The rows on ``dev``, contiguous, in their own dtype (fp16 / fp32; others, fp64 included, become fp32)."""
    x = torch.as_tensor(x)
    if x.dtype not in (torch.float16, torch.float32):
        x = x.to(dev, torch.float32)   # fp64 rows are rounded to fp32 here
    return x.to(dev).contiguous()


class RowPasses:
    """The engine's row passes over rows of width ``d`` on ``device`` in arithmetic ``arith``. Each method runs its pass
    over all the rows of ``x`` (fp16 or fp32 [B, d], contiguous, on ``device``) in ``call_rows(d)``-row calls on the
    current stream, with the rows shifted by ``shift`` (fp32 [d]); outputs accumulate as the engine's do. One workspace,
    grown to the largest call's need, serves every call; the range flag collects every call's f16f8 range check."""

    def __init__(self, d: int, device: torch.device, arith: str):
        self.d, self.device, self.code = int(d), device, _lib.arith_code(arith)
        self.flag = torch.zeros(1, dtype=torch.int32, device=device)
        self._ws, self._ws_ptr, self._ws_bytes = None, 0, 0

    def check_flag(self, what: str):
        if int(self.flag.item()):
            raise ValueError(f"{what} hold a value the f16f8 arithmetic's fp16 plane cannot (|v| >= 65520 or NaN): use "
                             f"arith='bf16x3' or 'auto'")

    def _calls(self, x, query: str, *sizes):
        """Per call over the rows of ``x``: (start, end, the call's leading arguments x, x_is_half, B, d, and its
        trailing ones workspace, workspace_bytes, stream). ``query(*sizes, B)`` sizes the workspace."""
        self.lib = _lib.load()
        cut = cuts(x.shape[0], self.d)
        need = max(getattr(self.lib, query)(*sizes, e - s) for s, e in cut)
        if need > self._ws_bytes:
            self._ws = None
            self._ws, self._ws_ptr = _lib.workspace(need, self.device, query)
            self._ws_bytes = need
        tail = (self._ws_ptr, self._ws_bytes, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        half = int(x.dtype == torch.float16)
        return [(s, e, (x[s:e].data_ptr(), half, e - s, self.d), tail) for s, e in cut]

    def second_moments(self, x, shift, col_sum, gram):
        """col_sum += sum of x - shift, gram += (x - shift)^T (x - shift) (fp64)."""
        for _, _, rows, ws in self._calls(x, "sce_second_moments_workspace_bytes", self.d):
            _lib.check(self.lib.sce_second_moments(*rows, shift.data_ptr(), self.code, col_sum.data_ptr(),
                                                   gram.data_ptr(), self.flag.data_ptr(), *ws), "sce_second_moments")

    def ica_pass(self, x, shift, unmix, alpha, g_sum, gx):
        """FastICA's data pass with unmix [n, d] (fp32): g_sum += sum alpha (1 - t^2), gx += t^T (x - shift)."""
        n = unmix.shape[0]
        for _, _, rows, ws in self._calls(x, "sce_ica_pass_workspace_bytes", self.d, n):
            _lib.check(self.lib.sce_ica_pass(*rows, shift.data_ptr(), unmix.data_ptr(), n, C.c_float(alpha), self.code,
                                             g_sum.data_ptr(), gx.data_ptr(), self.flag.data_ptr(), *ws), "sce_ica_pass")

    def nmf_project(self, x, shift, m, out, norms=None):
        """out[s:e] = max(x[s:e] - shift, 0) m^T (fp32) per call, adding the part norms to ``norms`` if given."""
        k = m.shape[0]
        for s, e, rows, ws in self._calls(x, "sce_nmf_project_workspace_bytes", self.d, k):
            _lib.check(self.lib.sce_nmf_project(*rows, shift.data_ptr(), m.data_ptr(), k, self.code, out[s:e].data_ptr(),
                                                None if norms is None else norms.data_ptr(), self.flag.data_ptr(), *ws),
                       "sce_nmf_project")

    def nmf_grams(self, x, shift, w, wtw, wtv):
        """wtw += w^T w, wtv += w^T max(x - shift, 0) (fp64) for the fp32 codes w [B, k] of the rows."""
        k = w.shape[1]
        for s, e, rows, ws in self._calls(x, "sce_nmf_grams_workspace_bytes", self.d, k):
            _lib.check(self.lib.sce_nmf_grams(*rows, shift.data_ptr(), w[s:e].data_ptr(), k, self.code, wtw.data_ptr(),
                                              wtv.data_ptr(), self.flag.data_ptr(), *ws), "sce_nmf_grams")

    def nmf_residual(self, x, shift, w, h, out):
        """out += ||max(x - shift, 0) - w h||^2 (fp64) for the fp32 codes w [B, k] and h [k, d]."""
        k = w.shape[1]
        for s, e, rows, ws in self._calls(x, "sce_nmf_residual_workspace_bytes", self.d):
            _lib.check(self.lib.sce_nmf_residual(*rows, shift.data_ptr(), w[s:e].data_ptr(), k, h.data_ptr(),
                                                 out.data_ptr(), *ws), "sce_nmf_residual")
