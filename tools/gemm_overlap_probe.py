"""How much of each split-operand GEMM of a config-2 training step is its epilogue, and what sharing A tiles saves.

Config 2: 16 tied SAEs, d = 512, n = 4096, batch 8192, f16f8 arithmetic, fp16-exact activations (bench.py's cfg2).
For each of the step's four GEMMs (encode, decode, dcode, weight gradient) it reports
  (a) engine_ms: the mean time of the engine's gemm_split_kernel launch inside step_batch, from torch.profiler with CUDA
      activities, in a run of its own;
  (b) main_loop_ms: the same kernel configuration at the same shapes with an epilogue that only reads the accumulators
      (build/gemm_overlap_probe, Makefile target `probe`), declaring the engine epilogue's staging bytes so that the
      stage ring is as deep; once in clusters of one CTA (each loads its own A tiles) and once in clusters of two along
      N (the pair shares each A tile by TMA multicast, as the engine launches decode and dW), in alternating order;
  (c) epilogue_bound_ms, encode and dcode only: the engine's kernel time for the same GEMM, measured as (a), at the same
      M, n and B but d = 64. Their K loop is then a single K block, so the time is bounded by the epilogue's per-tile
      throughput: where (c) is below (b), the epilogue keeps pace with the main loop at d = 512;
(d) tall_main_loop_ms, decode and the weight gradient only: (b) on 192-row output tiles (BM = kBMTall in
    sce_gemm.cuh), each launch right after the same one on 128-row tiles;
and the card's name, power limit and SM clock, read in the same run after each measurement. Beside them: (b) of encode
with 6 KB of epilogue staging per warp instead of 4 KB (one ring stage fewer, what staging the code's batch-major copies
through shared memory would cost), and the time and launches per step of transpose_batch_u8_kernel, the pass that makes
the batch-major copies of the 8-bit planes the epilogues do not write.
(a), (b) and (c) are taken in alternated rounds and their medians reported with the range. (a) minus (b) at the
cluster size the engine launches the GEMM in (2 for decode and dW, 1 for encode and dcode; the probe reports it) is the
time the epilogue adds; (b) at cluster 2 over (b) at cluster 1 is what a 25 % cut of the main loop's L2 operand reads
buys. (a) and (b) run on different operands (the engine's training data, hashed finite values), which alone can move
(b) against (a). Prints a table and one JSON line; --out DIR also writes it there.

    python tools/gemm_overlap_probe.py [--steps 20] [--reps 20] [--rounds 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

# epilogue functor in the kernel's name -> GEMM of the step
EPILOGUES = (("EpiEncodeT", "encode"), ("EpiDecodeT", "decode"), ("EpiDcodeT", "dcode"), ("EpiStoreF32", "dw"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), (v.strip() for v in out.split(","))))


class EngineRun:
    """A config-2 ensemble (at input dimension `d`, config 2's 512 by default), warmed up; `times()` profiles `steps`
    training steps and returns the mean device time of each GEMM launch of a step by epilogue (None where no launch of
    that epilogue was seen) and its launches per step."""

    def __init__(self, steps, d=None):
        import bench
        import sparse_coding_b200 as S

        M, d512, n, B, _ = bench.WORKLOADS["cfg2"]
        d = d or d512
        dev = torch.device("cuda", 0)
        sig = S.FunctionalTiedSAE
        self.ens = S.FunctionalEnsemble(bench.make_models(sig, M, d, n, seed=0), sig, S.adam, {"lr": 1e-3}, device=dev)
        self.pool = [x.to(dev) for x in bench.synth_batches(4, B, d, seed=1000)]
        self.steps = steps
        for i in range(5):
            self.ens.step_batch(self.pool[i % len(self.pool)])
        torch.cuda.synchronize()
        self.arith = self.ens.resolved_arith()

    def times(self):
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(self.steps):
                self.ens.step_batch(self.pool[i % len(self.pool)])
            torch.cuda.synchronize()
        sums = {g: [0.0, 0] for _, g in EPILOGUES}
        sums[TRANSPOSE] = [0.0, 0]
        for ev in prof.events():
            if TRANSPOSE in ev.name:
                sums[TRANSPOSE][0] += ev.device_time / 1e3
                sums[TRANSPOSE][1] += 1
            if "gemm_split_kernel" not in ev.name:
                continue
            for tag, g in EPILOGUES:
                if tag in ev.name:
                    sums[g][0] += ev.device_time / 1e3   # us -> ms
                    sums[g][1] += 1
                    break
        out = {g: (t / c if c else None, c / self.steps) for g, (t, c) in sums.items()}
        out[TRANSPOSE] = (sums[TRANSPOSE][0] / self.steps, sums[TRANSPOSE][1] / self.steps)   # per step, not per launch
        return out


TRANSPOSE = "transpose_batch_u8_kernel"
CLUSTERS = (1, 2)
EPILOGUE_BOUND_D = 64                 # input dimension of (c): one K block of the encode and dcode GEMMs
EPILOGUE_BOUND = ("encode", "dcode")  # the GEMMs (c) is reported for
TALL = ("decode", "dw")               # the GEMMs (d) is reported for


def main_loop_times(reps, clusters):
    exe = os.path.join(ROOT, "build", "gemm_overlap_probe")
    if not os.path.exists(exe):
        raise SystemExit(f"{exe} is missing: run `make probe` first")
    out = subprocess.run([exe, str(reps)] + [str(c) for c in clusters], capture_output=True, text=True,
                         check=True).stdout
    return {(r["gemm"], r["cluster"], r["bm"]): r for r in (json.loads(l) for l in out.splitlines() if l.startswith("{"))}


def fmt(v, width):
    return f"{v:{width}.3f}" if v is not None else f"{'-':>{width}s}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="profiled training steps per round")
    ap.add_argument("--reps", type=int, default=20, help="timed launches of each main-loop-only GEMM per round")
    ap.add_argument("--rounds", type=int, default=5, help="alternated rounds of (a) and (b); medians are reported")
    ap.add_argument("--out", default=None, help="directory for gemm_overlap_probe.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("the probe times kernels on cuda:0 and needs a GPU")
    info = card()
    run = EngineRun(args.steps)
    run_c = EngineRun(args.steps, d=EPILOGUE_BOUND_D)
    if run_c.arith != run.arith:
        raise SystemExit(f"d = {EPILOGUE_BOUND_D} runs {run_c.arith}, d = 512 {run.arith}: (c) would time another kernel")
    rounds = []
    for i in range(args.rounds):
        eng = run.times()
        clock_a = card()["clocks.sm"]
        ml = main_loop_times(args.reps, CLUSTERS if i % 2 == 0 else CLUSTERS[::-1])
        clock_b = card()["clocks.sm"]
        eb = run_c.times()
        clock_c = card()["clocks.sm"]
        rounds.append({"engine": eng, "main_loop": ml, "epilogue_bound": eb, "clock_after_engine": clock_a,
                       "clock_after_main_loop": clock_b, "clock_after_epilogue_bound": clock_c})

    def med(v):
        v = sorted(x for x in v if x is not None)
        return v[len(v) // 2] if v else None

    print(f"{info['name']}, power limit {info['power.limit']}, max SM clock {info['clocks.max.sm']}; SM clock read "
          f"after each round's (a), (b) and (c): "
          + ", ".join(f"{r['clock_after_engine']} / {r['clock_after_main_loop']} / {r['clock_after_epilogue_bound']}"
                      for r in rounds))
    print(f"medians of {args.rounds} rounds (min-max in brackets)")
    print(f"{'gemm':8s} {'launches/step':>13s} {'engine ms':>10s} {'':15s} {'main loop ms, cluster 1':>24s} {'':15s} "
          f"{'cluster 2':>10s} {'':15s} {'c2 / c1':>8s} {'epilogue ms':>12s} {'d=64 ms':>8s} {'':15s}"
          f"  (epilogue: (a) against the main loop at the engine's cluster size; d=64: (c))")
    rows = []
    for _, g in EPILOGUES:
        a = [r["engine"][g][0] for r in rounds]
        b = {c: [r["main_loop"][(g, c, 128)]["main_loop_ms"] for r in rounds] for c in CLUSTERS}
        tall = {c: [r["main_loop"][(g, c, 192)]["main_loop_ms"] for r in rounds] for c in CLUSTERS} if g in TALL else None
        per_step = rounds[0]["engine"][g][1]
        ma, mb1, mb2 = med(a), med(b[1]), med(b[2])
        ec = rounds[0]["main_loop"][(g, 1, 128)]["engine_cluster"]   # the cluster size the engine launches this GEMM in
        mbe = mb2 if ec == 2 else mb1
        av = [x for x in a if x is not None]
        cv = [r["epilogue_bound"][g][0] for r in rounds] if g in EPILOGUE_BOUND else []
        mc = med(cv)
        rows.append({"epilogue_bound_ms": mc, "epilogue_bound_ms_rounds": cv, "gemm": g, "launches_per_step": per_step, "engine_cluster": ec, "engine_ms": ma,
                     "main_loop_ms": mbe, "main_loop_ms_rounds": b[ec], "main_loop_ms_cluster1": mb1,
                     "main_loop_ms_cluster2": mb2, "main_loop_ms_cluster1_rounds": b[1],
                     "main_loop_ms_cluster2_rounds": b[2], "engine_ms_rounds": a,
                     "epilogue_ms": None if ma is None else ma - mbe,
                     "stages": rounds[0]["main_loop"][(g, 1, 128)]["stages"], "tiles": rounds[0]["main_loop"][(g, 1, 128)]["tiles"]})
        if tall:
            rows[-1].update({"tall_main_loop_ms_cluster1": med(tall[1]), "tall_main_loop_ms_cluster2": med(tall[2]),
                             "tall_main_loop_ms_cluster1_rounds": tall[1], "tall_main_loop_ms_cluster2_rounds": tall[2],
                             "tall_stages": rounds[0]["main_loop"][(g, 1, 192)]["stages"],
                             "tall_tiles": rounds[0]["main_loop"][(g, 1, 192)]["tiles"]})
        ra = f"[{min(av):.3f}-{max(av):.3f}]" if av else ""
        r1, r2 = f"[{min(b[1]):.3f}-{max(b[1]):.3f}]", f"[{min(b[2]):.3f}-{max(b[2]):.3f}]"
        cvv = [x for x in cv if x is not None]
        rc = f"[{min(cvv):.3f}-{max(cvv):.3f}]" if cvv else ""
        print(f"{g:8s} {per_step:13.1f} {fmt(ma, 10)} {ra:15s} {mb1:24.3f} {r1:15s} {mb2:10.3f} {r2:15s} "
              f"{mb2 / mb1:8.3f} {fmt(None if ma is None else ma - mbe, 12)} {fmt(mc, 8)} {rc:15s}")
    tr = [r["engine"][TRANSPOSE][0] for r in rounds]
    tr_launches = rounds[0]["engine"][TRANSPOSE][1]
    e6 = [r["main_loop"][("encode_6k", 1, 128)]["main_loop_ms"] for r in rounds]
    e6_stages = rounds[0]["main_loop"][("encode_6k", 1, 128)]["stages"]
    print(f"encode main loop with 6 KB staging per warp ({e6_stages} stages), cluster 1: {med(e6):.3f} "
          f"[{min(e6):.3f}-{max(e6):.3f}] ms")
    for row in rows:
        if "tall_main_loop_ms_cluster1" not in row:
            continue
        for c in CLUSTERS:
            t, t128 = row[f"tall_main_loop_ms_cluster{c}_rounds"], row[f"main_loop_ms_cluster{c}_rounds"]
            print(f"{row['gemm']} main loop, 192-row tiles ({row['tall_stages']} stages, {row['tall_tiles']} tiles), cluster {c}: "
                  f"{med(t):.3f} [{min(t):.3f}-{max(t):.3f}] ms, {med(t) / med(t128):.3f} x the 128-row tiles")
    print(f"{TRANSPOSE}: {med(tr):.3f} [{min(tr):.3f}-{max(tr):.3f}] ms per step, {tr_launches:.1f} launches per step")
    res = {"card": info, "encode_6k_main_loop_ms": med(e6), "encode_6k_main_loop_ms_rounds": e6,
           "encode_6k_stages": e6_stages, "transpose_ms_per_step": med(tr), "transpose_ms_per_step_rounds": tr,
           "transpose_launches_per_step": tr_launches, "arith": run.arith, "epilogue_bound_d": EPILOGUE_BOUND_D, "rounds": [{k: v for k, v in r.items() if k.startswith("clock")} for r in rounds], "gemms": rows}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gemm_overlap_probe.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
