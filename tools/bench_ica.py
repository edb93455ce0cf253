#!/usr/bin/env python
"""ICAEncoder fits on the engine against the same FastICA update as plain op sequences on the same GPU, and sklearn.
  ica_cfg2: d = 512, one 2^21-row fp16 chunk resident on the device (config 2's width)
  ica_cfg5: d = 2048, 2^21 rows (config 5's width)

    python tools/bench_ica.py --workload ica_cfg2|ica_cfg5 [--steps K --warmup W]

Prints one JSON line. Per arithmetic: CUDA-event ms of one engine pass over the chunk (sce_ica_pass in the fit's calls),
of the d x d fp64 update (gx Kw^T, the eigh-based symmetric decorrelation, lim), ms per iteration from fits of 1 and
1 + ITERS iterations ((t - t1) / ITERS), ms per fit at ITERS iterations (tol = 0: standardisation, whitening and the
read-out included), algorithmic TFLOP/s of a pass (4 N d n) and the pass's deviation from fp64, ||gx - gx64||_F /
||gx64||_F. Comparators: the same pass as an fp32 op sequence with TF32 off and on, and in fp64 (chunks of 65536 rows);
sklearn FastICA on the host over a subsample, per iteration, scaled to the chunk ("scaled": true), when sklearn can be
imported. The card name and power limit are read in the same call. Writes nothing to disk."""
import argparse
import ctypes as C
import json
import os
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_metrics import card_info, setup, timed  # noqa: E402

WORKLOADS = {"ica_cfg2": 512, "ica_cfg5": 2048}
N_ROWS = 1 << 21
CHUNK = 1 << 16
ITERS = 10


def chunk_rows(N, d, dev, seed=0):
    """[N, d] fp16 rows: Laplace sources mixed by a seeded matrix around a non-zero offset, generated on the device."""
    g = torch.Generator(device=dev).manual_seed(seed)
    A = 0.3 * torch.randn(d, d, generator=g, device=dev) / d ** 0.5 + torch.eye(d, device=dev)
    mu = 2.0 * torch.randn(d, generator=g, device=dev)
    x = torch.empty(N, d, dtype=torch.float16, device=dev)
    for s in range(0, N, CHUNK):
        u = (torch.rand(min(CHUNK, N - s), d, generator=g, device=dev) - 0.5).clamp_(min=-0.4999999)   # log1p(-1) = -inf
        x[s:s + CHUNK] = (mu + (-torch.sign(u) * torch.log1p(-2 * u.abs())) @ A.T).half()
    return x


def op_pass(x, shift, unmix, dtype):
    """g_sum, gx of one pass as a torch op sequence in ``dtype``, in chunks."""
    n, d = unmix.shape
    g_sum = torch.zeros(n, dtype=torch.float64, device=x.device)
    gx = torch.zeros(n, d, dtype=dtype, device=x.device)
    w = unmix.to(dtype)
    for s in range(0, x.shape[0], CHUNK):
        v = x[s:s + CHUNK].to(dtype) - shift.to(dtype)
        t = torch.tanh(v @ w.T)
        g_sum += (1 - t * t).sum(0, dtype=torch.float64)
        gx += t.T @ v
    return g_sum, gx.double()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="ica_cfg2")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sklearn-rows", type=int, default=0, help="host subsample (default: 16384 at d = 512, 4096 above)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_ica.py needs a CUDA device (the engine has no CPU path)")
    dev, K, W = setup(args)
    from sparse_coding_b200 import _lib
    from sparse_coding_b200.ica import ICAEncoder, _sym_decorrelation
    from sparse_coding_b200._rowpass import call_rows
    d, N = WORKLOADS[args.workload], N_ROWS
    x = chunk_rows(N, d, dev)
    flops = 4.0 * N * d * d
    out = {"workload": args.workload, "d": d, "rows": N, "input": "fp16, resident", "iters": ITERS, "engine": {},
           "comparators": {}}
    rs = np.random.RandomState(0)
    w_init = rs.normal(size=(d, d))
    shift = x[:CHUNK].float().mean(0).contiguous()
    unmix = (torch.from_numpy(rs.normal(size=(d, d))).float().to(dev) / d ** 0.5).contiguous()
    ref64 = op_pass(x, shift, unmix, torch.float64)
    lib = _lib.load()
    step = call_rows(d)
    ws, ptr = _lib.workspace(lib.sce_ica_pass_workspace_bytes(d, d, step), dev, "sce_ica_pass_workspace_bytes")
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    warnings.simplefilter("ignore")

    for arith in ("bf16x3", "f16f8"):
        print(f"{args.workload}: engine, {arith}", file=sys.stderr, flush=True)
        code = _lib.arith_code(arith)

        def engine_pass():
            g_sum = torch.zeros(d, dtype=torch.float64, device=dev)
            gx = torch.zeros(d, d, dtype=torch.float64, device=dev)
            for s in range(0, N, step):
                _lib.check(lib.sce_ica_pass(x[s].data_ptr(), 1, min(step, N - s), d, shift.data_ptr(), unmix.data_ptr(),
                                            d, C.c_float(1.0), code, g_sum.data_ptr(), gx.data_ptr(), None, ptr,
                                            ws.numel() - 1024, stream), "sce_ica_pass")
            return g_sum, gx
        ms_pass, (g_sum, gx) = timed(engine_pass, K, W)
        Wm = _sym_decorrelation(torch.from_numpy(w_init).to(dev))
        Kw = torch.eye(d, dtype=torch.float64, device=dev)

        def update():
            W1 = _sym_decorrelation(gx @ Kw.T / N - (g_sum / N)[:, None] * Wm)
            return float(((W1 * Wm).sum(dim=1).abs() - 1).abs().max())
        ms_dd, _ = timed(update, K, W)

        def fit(iters):
            return lambda: ICAEncoder(d, device=dev, arith=arith, max_iter=iters, tol=0.0, w_init=w_init).fit(x)
        ms1, _ = timed(fit(1), K, W)
        ms_fit, _ = timed(fit(1 + ITERS), K, W)
        out["engine"][arith] = {
            "pass_ms": ms_pass, "dd_update_ms": ms_dd, "ms_per_iter": (ms_fit - ms1) / ITERS,
            "fit_ms": ms_fit - (ms_fit - ms1) / ITERS, "pass_tflops": flops / ms_pass * 1e-9,
            "gx_dev": float((gx - ref64[1]).norm() / ref64[1].norm()),
            "g_sum_dev": float((g_sum - ref64[0]).norm() / ref64[0].norm())}

    print(f"{args.workload}: op sequences", file=sys.stderr, flush=True)
    for name, tf32 in (("ops_fp32", False), ("ops_tf32", True)):
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        try:
            ms, (g_sum, gx) = timed(lambda: op_pass(x, shift, unmix, torch.float32), K, W)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
        out["comparators"][name] = {"pass_ms": ms, "pass_tflops": flops / ms * 1e-9,
                                    "gx_dev": float((gx - ref64[1]).norm() / ref64[1].norm())}
    ms, _ = timed(lambda: op_pass(x, shift, unmix, torch.float64), 1, 1)
    out["comparators"]["ops_fp64"] = {"pass_ms": ms, "pass_tflops": flops / ms * 1e-9, "gx_dev": 0.0}

    try:
        from sklearn.decomposition import FastICA
        from sklearn.preprocessing import StandardScaler
    except ImportError:
        out["comparators"]["sklearn"] = {"skipped": "sklearn is not installed"}
    else:
        print(f"{args.workload}: sklearn", file=sys.stderr, flush=True)
        rows = args.sklearn_rows or (16384 if d <= 512 else 4096)
        sub = StandardScaler().fit_transform(x[:rows].double().cpu().numpy())
        per = {}
        for iters in (1, 3):
            t0 = time.perf_counter()
            FastICA(max_iter=iters, tol=0.0, w_init=w_init).fit(sub)
            per[iters] = time.perf_counter() - t0
        it_ms = (per[3] - per[1]) / 2 * 1e3 * (N / rows)
        out["comparators"]["sklearn"] = {"ms_per_iter": it_ms, "scaled": True, "timed_rows": rows,
                                         "threads": torch.get_num_threads()}
    name, limit = card_info(dev.index)
    out["gpu"], out["power_limit_w"] = name, limit
    print(json.dumps(out))


if __name__ == "__main__":
    main()
