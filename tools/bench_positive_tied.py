#!/usr/bin/env python
"""Step time of FunctionalPositiveTiedSAE (non-negative tied dictionary on x + 0.18) against FunctionalTiedSAE with the
same bias decay, at two shapes: the reference's run_positive sweep (9 models, d = n = 2048, B = 2048, L1 = {0} and
logspace(-5, -3.5, 8), bias decay 0.01) and config 2's (16 models, d = 512, n = 4096, B = 8192, L1 = logspace(-4, -2,
16)); and of the comparator a user has without the engine: the reference's vmap(grad(loss)) + Adam
(oracle.sae_oracle.RefPortEnsemble with the restated positive-tied loss) on the same GPU, in fp32 and with TF32.

    python tools/bench_positive_tied.py [--steps K --warmup W --rounds R --ref-steps S]

At each shape the engine signatures run alternately in one process (FunctionalTiedSAE also a second time, fed x + 0.18,
which is not fp16-exact, to show what inexact input alone costs), R rounds of K timed steps each (after W
warm-up steps), on the same seeded fp16-representable MLP-like activations (GELU of a sparse mixture). Times are
CUDA-event milliseconds per step; the per-phase split comes from profile_begin / profile_end on one extra round. Prints
one JSON line with the card name and power limit read in the same run. Writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {   # name: (M, d, n, B, l1 grid)
    "catalogue": (9, 2048, 2048, 2048, [0.0] + np.logspace(-5, -3.5, 8).tolist()),
    "cfg2": (16, 512, 4096, 8192, np.logspace(-4, -2, 16).tolist()),
}
BIAS_DECAY = 0.01


def card_info(index):
    """(name, power limit in W) of the GPU, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().split(",")[:2]]
        return name, float(limit)
    except Exception:
        return torch.cuda.get_device_name(index), None


def batches(count, B, d, seed):
    """`count` seeded [B, d] batches of fp16-representable MLP-like activations."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    feats = torch.randn(4096, d, generator=gen, device="cuda")
    feats /= feats.norm(dim=-1, keepdim=True)
    out = []
    for _ in range(count):
        codes = (torch.rand(B, 4096, generator=gen, device="cuda") < 0.005).float() * \
            torch.rand(B, 4096, generator=gen, device="cuda")
        z = 3.0 * codes @ feats + 0.5 * torch.randn(B, d, generator=gen, device="cuda")
        out.append(torch.nn.functional.gelu(z).half().float())
    return out


def models(S, kind, shape, seed):
    M, d, n, B, l1s = SHAPES[shape]
    torch.manual_seed(seed)
    if kind == "positive_tied":
        return [S.FunctionalPositiveTiedSAE.init(d, n, a, BIAS_DECAY) for a in l1s]
    return [S.FunctionalTiedSAE.init(d, n, a, bias_decay=BIAS_DECAY) for a in l1s]


def timed(fn, xs, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(xs[i % len(xs)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_shape(S, O, PT, shape, args):
    M, d, n, B, _ = SHAPES[shape]
    xs = batches(4, B, d, 0)
    # "tied_inexact": FunctionalTiedSAE fed x + 0.18 itself, which is no longer fp16-exact, as the positive-tied step
    # sees it: it separates the cost of inexact input (the f16f8 residual cross terms of x run) from that of the rest
    shifted = [x + 0.18 for x in xs]
    sigs = {"tied": S.FunctionalTiedSAE, "tied_inexact": S.FunctionalTiedSAE, "positive_tied": S.FunctionalPositiveTiedSAE}
    data = {"tied": xs, "tied_inexact": shifted, "positive_tied": xs}
    ens = {k: S.FunctionalEnsemble(models(S, "tied" if k == "tied_inexact" else k, shape, 0), sig, S.adam, {"lr": 1e-3},
                                   device="cuda") for k, sig in sigs.items()}
    for k, e in ens.items():
        timed(e.step_batch, data[k], args.warmup)
    ms = {k: [] for k in ens}
    for _ in range(args.rounds):
        for k, e in ens.items():
            ms[k].append(timed(e.step_batch, data[k], args.steps))
    phases = {}
    for k, e in ens.items():
        e.profile_begin()
        timed(e.step_batch, data[k], min(args.steps, 64))
        p = e.profile_end()
        phases[k] = {ph: round(v / p["steps"], 4) for ph, v in p.items() if ph != "steps"}
    med = {k: round(float(np.median(vs)), 4) for k, vs in ms.items()}
    out = {"M": M, "d": d, "n": n, "B": B, "arith": ens["positive_tied"].resolved_arith(),
           "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in ms.items()}, "ms_per_step_median": med,
           "positive_over_tied": round(med["positive_tied"] / med["tied"], 4),
           "positive_over_tied_inexact": round(med["positive_tied"] / med["tied_inexact"], 4), "phase_ms_per_step": phases}
    del ens
    torch.cuda.empty_cache()
    if args.ref_steps > 0:
        ref_ms = {}
        for label, tf32 in (("ref_fp32", False), ("ref_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms_ = [({k: v.cuda() for k, v in p.items()}, {k: v.cuda() for k, v in b.items()})
                   for p, b in models(S, "positive_tied", shape, 0)]
            ref = O.RefPortEnsemble(ms_, PT.sig_loss_positive_tied, lr=1e-3)
            timed(ref.step_batch, xs, 1)
            ref_ms[label] = round(timed(ref.step_batch, xs, args.ref_steps), 3)
            del ref, ms_
            torch.cuda.empty_cache()
        torch.backends.cuda.matmul.allow_tf32 = False
        out["ref_ms_per_step"] = ref_ms
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ref-steps", type=int, default=3, help="timed steps of each reference comparator (0: skip them)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_positive_tied.py needs a CUDA device (the engine has no CPU path)")
    import sparse_coding_b200 as S
    from oracle import positive_tied_oracle as PT
    from oracle import sae_oracle as O
    torch.cuda.set_device(0)
    name, limit = card_info(0)
    out = {"workload": "positive_tied", "gpu": name, "power_limit_w": limit, "bias_decay": BIAS_DECAY,
           "rounds": args.rounds, "steps_per_round": args.steps}
    for shape in SHAPES:
        out[shape] = bench_shape(S, O, PT, shape, args)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
