"""Cost of dead-feature tracking and resampling, and what resampling does to a synthetic training run.

  python tools/bench_resample.py [--out DIR]

1. Config 2 (16 tied SAEs, d = 512, n = 4096, B = 8192, f16f8): step time without a window and with one open
   (n_worst = n), three alternated runs of 20 timed steps each after warm-up; the time of one resample_dead_features
   call. Config 5 (1 tied SAE, d = 2048, n = 32768, B = 4096): one run each.
2. Synthetic data (SparseMixDataset, d = 256, 512 ground-truth features, 16 tied SAEs with n = 2048 and L1 =
   logspace(-3, -0.5)): train_on_chunks
   over 12 SyntheticChunks with and without resample_every = 2, then per model the dead fraction on a held-out batch
   and the MMCS of the ground truth to the learned dictionary (as tools/train_synthetic.py).
Prints one JSON line (card name and power limit included) and writes it to DIR/bench_resample.json."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import sparse_coding_b200 as S
from sparse_coding_b200.metrics import evaluate
from sparse_coding_b200.train_loop import train_on_chunks


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unknown ({e})"
    return q


def make(M, d, n, l1=(-4, -2)):
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(d, n, float(a)) for a in np.logspace(*l1, M)]
    return S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")


def timed_steps(ens, X, steps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        ens.step_batch(X)
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def step_costs(M, d, n, B, runs, steps=20):
    gen = torch.Generator(device="cuda").manual_seed(1)
    X = torch.randn(B, d, device="cuda", generator=gen).half().float()
    plain, tracked = make(M, d, n), make(M, d, n)
    tracked.track_dead_features()
    for e in (plain, tracked):
        for _ in range(5):
            e.step_batch(X)
    out = {"untracked_ms": [], "tracked_ms": []}
    for _ in range(runs):
        out["untracked_ms"].append(round(timed_steps(plain, X, steps), 4))
        out["tracked_ms"].append(round(timed_steps(tracked, X, steps), 4))
    out["arith"] = tracked.resolved_arith()
    out["launches_untracked"] = plain.gpu_launches_last_call()
    torch.cuda.synchronize()
    t0 = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    t0[0].record()
    r = tracked.resample_dead_features()
    t0[1].record()
    torch.cuda.synchronize()
    out["resample_ms"] = round(t0[0].elapsed_time(t0[1]), 4)
    out["resample_n_dead"] = r["n_dead"].tolist()
    out["overhead_pct"] = round(100 * (np.median(out["tracked_ms"]) / np.median(out["untracked_ms"]) - 1), 2)
    del plain, tracked
    torch.cuda.empty_cache()
    return out


SYNTH_L1 = (-3, -0.5)   # strong penalties at the top of the range, where features die


def synthetic(resample_every, n_chunks=12):
    d, n_gt, n, M, bs = 256, 512, 2048, 16, 2048
    np.random.seed(0)
    gen = S.SparseMixDataset(d, n_gt, 4 * bs, 8, 0.99, 0.0, "cuda", sparse_component_covariance=torch.eye(n_gt, device="cuda"),
                             t_type=torch.float16, seed=123)
    truth = gen.sparse_component_dict.float()
    truth = truth / truth.norm(dim=-1, keepdim=True)
    ens = make(M, d, n, SYNTH_L1)
    chunks = S.SyntheticChunks(gen, n_chunks, 1 << 16)
    replaced = []
    with tempfile.TemporaryDirectory() as tmp:
        train_on_chunks(ens, {"device": "cuda"}, None, tmp, bs, [], ["l1_alpha"], chunks=chunks,
                        resample_every=resample_every,
                        on_resample=lambda i, c, e, r: replaced.append(int(r["n_replaced"].sum())))
    held = chunks.chunk(n_chunks - 1)[: 4 * bs].float()
    ev = evaluate(ens, held, n_ever_active=True)
    W = ens.params["encoder"] / ens.params["encoder"].norm(dim=-1, keepdim=True)
    mmcs = torch.stack([(truth @ W[m].T).max(dim=-1).values.mean() for m in range(M)])
    return {"resample_every": resample_every, "chunks": n_chunks, "rows_per_chunk": 1 << 16,
            "frac_dead": [round(float(v), 3) for v in ev["frac_dead"]],
            "mmcs": [round(float(v), 3) for v in mmcs], "replaced_per_resample": replaced}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--synthetic-only", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resample measures on the GPU"
    line = {"card": card(), "synthetic_l1_alpha": [float(a) for a in np.logspace(*SYNTH_L1, 16)]}
    if not args.synthetic_only:
        line["cfg2"] = step_costs(16, 512, 4096, 8192, args.runs)
        line["cfg5"] = step_costs(1, 2048, 32768, 4096, 1)
    line["synthetic"] = [synthetic(0), synthetic(2)]
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_resample.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
