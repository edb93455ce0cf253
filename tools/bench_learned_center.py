#!/usr/bin/env python
"""Step time of FunctionalTiedCenteredSAE (learned centre) against FunctionalTiedSAE at config 2's shape (16 models,
d = 512, n = 4096, B = 8192, L1 = logspace(-4, -2, 16)), and of the comparator a user has without the engine: the
reference's vmap(grad(loss)) + Adam (oracle.sae_oracle.RefPortEnsemble) on the same GPU, in fp32 and with TF32.

    python tools/bench_learned_center.py [--steps K --warmup W --rounds R --ref-steps S]

The two engine signatures run alternately in one process, R rounds of K timed steps each (after W warm-up steps), on
the same seeded fp16-representable activations with a non-zero column mean. Times are CUDA-event milliseconds per step;
the per-phase split comes from profile_begin / profile_end on one extra round. Prints one JSON line with the card name
and power limit read in the same run. Writes nothing to disk."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

M, D, N, B = 16, 512, 4096, 8192


def card_info(index):
    """(name, power limit in W) of the GPU, read in the same run as the measurement."""
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in r.stdout.strip().split(",")[:2]]
        return name, float(limit)
    except Exception:
        return torch.cuda.get_device_name(index), None


def batches(count, seed):
    """`count` seeded [B, D] batches of fp16-representable sparse-mixture activations offset from the origin."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    feats = torch.randn(2048, D, generator=gen, device="cuda")
    feats /= feats.norm(dim=-1, keepdim=True)
    mu = 0.5 * torch.randn(D, generator=gen, device="cuda")
    out = []
    for _ in range(count):
        codes = (torch.rand(B, 2048, generator=gen, device="cuda") < 0.01).float() * \
            torch.rand(B, 2048, generator=gen, device="cuda")
        out.append((codes @ feats + 0.05 * torch.randn(B, D, generator=gen, device="cuda") + mu).half().float())
    return out


def models(sig, seed):
    torch.manual_seed(seed)
    return [sig.init(D, N, float(a)) for a in np.logspace(-4, -2, M)]


def timed(fn, xs, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(xs[i % len(xs)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ref-steps", type=int, default=3, help="timed steps of each reference comparator (0: skip them)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_learned_center.py needs a CUDA device (the engine has no CPU path)")
    import sparse_coding_b200 as S
    from oracle import learned_center_oracle as LC
    from oracle import sae_oracle as O
    torch.cuda.set_device(0)
    name, limit = card_info(0)
    xs = batches(4, 0)
    ens = {"tied": S.FunctionalEnsemble(models(S.FunctionalTiedSAE, 0), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3},
                                        device="cuda"),
           "learned_center": S.FunctionalEnsemble(models(S.FunctionalTiedCenteredSAE, 0), S.FunctionalTiedCenteredSAE,
                                                  S.adam, {"lr": 1e-3}, device="cuda")}
    for e in ens.values():
        timed(e.step_batch, xs, args.warmup)
    ms = {k: [] for k in ens}
    for _ in range(args.rounds):
        for k, e in ens.items():
            ms[k].append(timed(e.step_batch, xs, args.steps))
    phases = {}
    for k, e in ens.items():
        e.profile_begin()
        timed(e.step_batch, xs, min(args.steps, 64))
        p = e.profile_end()
        phases[k] = {ph: round(v / p["steps"], 4) for ph, v in p.items() if ph != "steps"}
    out = {"workload": "learned_center_cfg2", "M": M, "d": D, "n": N, "B": B, "gpu": name, "power_limit_w": limit,
           "arith": ens["learned_center"].resolved_arith(), "rounds": args.rounds, "steps_per_round": args.steps,
           "ms_per_step": {k: [round(v, 4) for v in vs] for k, vs in ms.items()},
           "ms_per_step_median": {k: round(float(np.median(vs)), 4) for k, vs in ms.items()},
           "phase_ms_per_step": phases}
    out["learned_center_over_tied"] = round(out["ms_per_step_median"]["learned_center"] /
                                            out["ms_per_step_median"]["tied"], 4)
    del ens
    torch.cuda.empty_cache()
    if args.ref_steps > 0:
        ref_ms = {}
        for label, tf32 in (("ref_fp32", False), ("ref_tf32", True)):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms_ = [({k: v.cuda() for k, v in p.items()}, {k: v.cuda() for k, v in b.items()})
                   for p, b in models(S.FunctionalTiedCenteredSAE, 0)]
            ref = O.RefPortEnsemble(ms_, LC.sig_loss_tied_learned_center, lr=1e-3)
            timed(ref.step_batch, xs, 1)
            ref_ms[label] = round(timed(ref.step_batch, xs, args.ref_steps), 3)
            del ref, ms_
            torch.cuda.empty_cache()
        torch.backends.cuda.matmul.allow_tf32 = False
        out["ref_ms_per_step"] = ref_ms
    print(json.dumps(out))


if __name__ == "__main__":
    main()
