"""Synthetic-chunk generation rate: ms per 2**21-row chunk (big_sweep's chunk at d = 512, 2 GB) made by
SyntheticChunks on the GPU, for the reference's synthetic workloads, against the reference's per-send op sequence
(random_dataset.py:119-139, 191-245: MultivariateNormal draw, ndtr, three dense [4096, n_gt] uniforms, zero-row fill,
fp32 GEMM, noise) restated in torch on the same GPU, once kept on the device and once with big_sweep's per-send
.cpu() into a host fp32 chunk (big_sweep.py:228-237). The comparator is timed over --ref-sends sends and scaled to the
512 sends of a chunk. Prints one JSON line; the card and its power limit are read in the same run.

  python tools/bench_synth.py --steps 5 --warmup 1

Workloads: run_dict_ratio (big_sweep_experiments.py:580-617: n_gt 2048, 100 non-zeros, decay 0.996, no noise) and
synthetic_test (:814-848: n_gt 1024 / 2048 x 10 / 50 / 100 non-zeros, noise 0.1, decay 1.0), all d = 512, fp16 rows,
identity covariance, generator batch 4096. gather_bytes counts what the gather reads from L2: rows x mean active
components x d x 4."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

D, GEN_BATCH, CHUNK_ROWS = 512, 4096, 1 << 21
WORKLOADS = [("run_dict_ratio", 2048, 100, 0.996, 0.0)] + [
    (f"synthetic_test_{n}_{k}", n, k, 1.0, 0.1) for k in (10, 50, 100) for n in (1024, 2048)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def reference_send(gen, dev):
    """One SparseMixDataset.send of the reference, op for op, on the device."""
    n = gen.n_sparse_components
    mvn = torch.distributions.MultivariateNormal(torch.zeros(n, device=dev), covariance_matrix=gen.sparse_component_covariance)
    z = mvn.sample()
    normal = torch.distributions.Normal(torch.tensor([0.0], device=dev), torch.tensor([1.0], device=dev))
    p = normal.cdf(z.squeeze()) * gen.sparse_component_probs
    p *= gen.frac_nonzero / torch.mean(p)
    thresh = torch.rand(GEN_BATCH, n, device=dev)
    values = torch.rand(GEN_BATCH, n, device=dev)
    codes = torch.where(thresh <= p, values, torch.zeros_like(z))
    zero = (codes.count_nonzero(dim=1) == 0).nonzero()[:, 0]
    codes[zero, torch.randint(low=0, high=n, size=(zero.shape[0],)).to(dev)] = 1.0
    strengths = torch.rand(GEN_BATCH, n, device=dev)
    x = (codes * strengths) @ gen.sparse_component_dict
    noise = torch.distributions.MultivariateNormal(torch.zeros(D, device=dev), covariance_matrix=gen.noise_covariance)
    x = x + noise.sample(torch.Size([GEN_BATCH])) * gen.noise_magnitude_scale
    return x.to(gen.t_type)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--ref-sends", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_synth measures the GPU generator: no CUDA device")
    import sparse_coding_b200 as S
    from sparse_coding_b200.synthetic import synth_rows
    dev = torch.device("cuda", 0)
    name, power = card()
    sends = CHUNK_ROWS // GEN_BATCH
    results = []
    for wl, n_gt, nnz, decay, noise in WORKLOADS:
        np.random.seed(0)
        gen = S.SparseMixDataset(D, n_gt, GEN_BATCH, nnz, decay, noise, dev, t_type=torch.float16, seed=1,
                                 sparse_component_covariance=torch.eye(n_gt, device=dev))
        chunks = S.SyntheticChunks(gen, 1, CHUNK_ROWS)
        ms = timed(lambda: chunks.chunk(0), args.steps, args.warmup)
        _, row_nnz, _, _ = synth_rows(gen.sparse_component_dict, gen._group_probs(0, 16), GEN_BATCH, 0, 16 * GEN_BATCH,
                                      gen.seed, True, noise, torch.float16)
        active = float(row_nnz.double().mean())
        gather_bytes = CHUNK_ROWS * active * D * 4
        ref_dev = timed(lambda: reference_send(gen, dev), args.ref_sends, 2) * sends
        host = torch.zeros(GEN_BATCH * args.ref_sends, D, dtype=torch.float32)

        def ref_cpu():
            for j in range(args.ref_sends):
                host[j * GEN_BATCH:(j + 1) * GEN_BATCH] = reference_send(gen, dev).cpu()

        ref_host = timed(ref_cpu, 1, 1) / args.ref_sends * sends
        results.append({"workload": wl, "n_gt": n_gt, "nonzeros": nnz, "decay": decay, "noise": noise,
                        "ms_per_chunk": round(ms, 3), "rows_per_s": round(CHUNK_ROWS / ms * 1e3),
                        "mean_active": round(active, 2), "gather_bytes": int(gather_bytes),
                        "gather_GB_per_s": round(gather_bytes / ms / 1e6, 1),
                        "ref_device_ms_per_chunk": round(ref_dev, 1), "ref_host_ms_per_chunk": round(ref_host, 1),
                        "speedup_vs_ref_device": round(ref_dev / ms, 1), "speedup_vs_ref_host": round(ref_host / ms, 1)})
        del chunks, gen
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "synthetic_chunks", "card": name, "power_limit": power, "chunk_rows": CHUNK_ROWS,
                      "d": D, "steps": args.steps, "warmup": args.warmup, "ref_sends": args.ref_sends,
                      "workloads": results}))


if __name__ == "__main__":
    main()
