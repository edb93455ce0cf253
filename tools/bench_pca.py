#!/usr/bin/env python
"""BatchedPCA fits on the engine against the reference's op sequence and plain Gram products on the same GPU.
  pca_cfg2: d = 512, one 2^21-row fp16 chunk resident on the device (config 2's width)
  pca_cfg5: d = 2048, 2^21 rows (config 5's width)

    python tools/bench_pca.py --workload pca_cfg2|pca_cfg5 [--steps K --warmup W]

Prints one JSON line: per arithmetic, CUDA-event ms per fit of the whole chunk (shift pass included), rows/s and
algorithmic TFLOP/s (2 N d^2); the comparators with their times: the reference's train_batch op sequence (an outer-
product tensor [B, d, d] per batch) at batch 500 and 5000 where the tensor fits, timed over a subset of batches and scaled
to the chunk ("scaled": true); X^T X in fp32 with TF32 off, with TF32 on, and in fp64 (chunks of 65536 rows). Each
result carries its deviation from fp64: ||C - C64||_F / ||C64||_F and max|mean - mean64| / max|mean64| (the reference's
on the rows of its timed subset). The card name and power limit are read in the same call. Writes nothing to disk."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_metrics import card_info, setup, timed  # noqa: E402

WORKLOADS = {"pca_cfg2": 512, "pca_cfg5": 2048}
N_ROWS = 1 << 21
CHUNK = 1 << 16


def chunk_rows(N, d, dev, seed=0):
    """[N, d] fp16 rows with a decaying spectrum around a non-zero mean, generated on the device."""
    g = torch.Generator(device=dev).manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(d, d, generator=g, device=dev))
    lam = 1.0 / (1.0 + torch.arange(d, device=dev, dtype=torch.float32))
    mu = 2.0 * torch.randn(d, generator=g, device=dev)
    x = torch.empty(N, d, dtype=torch.float16, device=dev)
    for s in range(0, N, CHUNK):
        z = torch.randn(min(CHUNK, N - s), d, generator=g, device=dev)
        x[s:s + CHUNK] = (mu + (z * lam.sqrt()) @ q.T).half()
    return x


def fp64_moments(x, rows=None):
    """(mean, cov) in fp64 over the first ``rows`` rows of x, in chunks."""
    N = x.shape[0] if rows is None else rows
    shift = x[: min(N, CHUNK)].double().mean(0)
    s1 = torch.zeros_like(shift)
    s2 = torch.zeros(x.shape[1], x.shape[1], dtype=torch.float64, device=x.device)
    for s in range(0, N, CHUNK):
        v = x[s:min(s + CHUNK, N)].double() - shift
        s1 += v.sum(0)
        s2 += v.T @ v
    return shift + s1 / N, (s2 - torch.outer(s1, s1) / N) / N


def naive_fp32(x):
    """The one-pass formula X^T X / N - mu mu^T in fp32, in chunks."""
    d = x.shape[1]
    g = torch.zeros(d, d, device=x.device)
    s1 = torch.zeros(d, device=x.device)
    for s in range(0, x.shape[0], CHUNK):
        v = x[s:s + CHUNK].float()
        g += v.T @ v
        s1 += v.sum(0)
    mu = s1 / x.shape[0]
    return mu, g / x.shape[0] - torch.outer(mu, mu)


def reference_ops(x, batch, n_batches):
    """The reference's train_batch op sequence (autoencoders/pca.py:54-64) over the first n_batches batches: the running
    mean, the batch's outer-product tensor [B, d, d] averaged over the batch, and the weighted merge, in fp32."""
    d = x.shape[1]
    mean = torch.zeros(d, device=x.device)
    cov = torch.zeros(d, d, device=x.device)
    n = 0
    for i in range(n_batches):
        a = x[i * batch:(i + 1) * batch].float()
        b = a.shape[0]
        corrected = a - mean[None]
        new_mean = mean + corrected.mean(0) * b / (n + b)
        upd = torch.einsum("bi,bj->bij", corrected, a - new_mean[None]).mean(0)
        cov = cov * (n / (n + b)) + upd * b / (n + b)
        mean = new_mean
        n += b
    return mean, cov


def deviation(mean, cov, ref):
    m64, c64 = ref
    return {"cov_dev": float((cov.double() - c64).norm() / c64.norm()),
            "mean_dev": float((mean.double() - m64).abs().max() / m64.abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=sorted(WORKLOADS), default="pca_cfg2")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_pca.py needs a CUDA device (the engine has no CPU path)")
    dev, K, W = setup(args)
    from sparse_coding_b200.pca import BatchedPCA
    d, N = WORKLOADS[args.workload], N_ROWS
    x = chunk_rows(N, d, dev)
    flops = 2.0 * N * d * d
    ref64 = fp64_moments(x)
    out = {"workload": args.workload, "d": d, "rows": N, "input": "fp16, resident", "engine": {}, "comparators": {}}

    for arith in ("bf16x3", "f16f8"):
        def fit():
            p = BatchedPCA(d, dev, arith=arith)
            p.train_batch(x)
            return p
        ms, p = timed(fit, K, W)
        out["engine"][arith] = {"ms": ms, "rows_per_s": N / ms * 1e3, "tflops": flops / ms * 1e-9,
                                **deviation(p.get_mean(), p._cov64(), ref64)}

    for name, tf32 in (("xtx_fp32", False), ("xtx_tf32", True)):
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        try:
            ms, (mu, cov) = timed(lambda: naive_fp32(x), K, W)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
        out["comparators"][name] = {"ms": ms, "tflops": flops / ms * 1e-9, **deviation(mu, cov, ref64)}
    ms, _ = timed(lambda: fp64_moments(x), 1, 1)
    out["comparators"]["xtx_fp64"] = {"ms": ms, "tflops": flops / ms * 1e-9, "cov_dev": 0.0, "mean_dev": 0.0}

    free = torch.cuda.mem_get_info(dev)[0]
    for batch in (500, 5000):
        if 3 * batch * d * d * 4 > free:          # the [B, d, d] tensor and its temporaries
            out["comparators"][f"reference_b{batch}"] = {"skipped": f"[{batch}, {d}, {d}] fp32 does not fit"}
            continue
        n_timed = max(2, min(N // batch, (1 << 14) // batch))
        ms, (mu, cov) = timed(lambda: reference_ops(x, batch, n_timed), 1, 1)
        full = ms * (N / (n_timed * batch))
        out["comparators"][f"reference_b{batch}"] = {
            "ms": full, "scaled": True, "timed_rows": n_timed * batch, "tflops": flops / full * 1e-9,
            **deviation(mu, cov, fp64_moments(x, n_timed * batch))}
    name, limit = card_info(dev.index)
    out["gpu"], out["power_limit_w"] = name, limit
    print(json.dumps(out))


if __name__ == "__main__":
    main()
