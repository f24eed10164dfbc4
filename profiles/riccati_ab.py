#!/usr/bin/env python3
"""Where the time of the Riccati backward pass `k_riccati_frag` (R) goes, on one GPU.

Alternates the default library with variants of riccati_frag.cu built with other flags (`--variant NAME=FLAGS`, e.g.
`minb7=-DTO_FRAG_MINB=7`, `stages3=-DTO_FRAG_STAGES=3`), `bench.py --gpus 1 --steps 20 --warmup 3` per library, workload and batch size,
with the card's name and power limit; prints the phase times R (backward), F (forward = pass 1), L (ladder = late passes), C1 + E1 and
the step time, and compares the `--dump-outputs` of every run of one workload and batch bitwise (the variants change scheduling, not
arithmetic).  `--batch` sweeps the batch size: at B = 528 every scheduler of the 132 SMs holds one warp (a lone sweep, dependent latency
only), at 3168 every resident warp slot of the default build is busy (one full wave), at 4096 a second, partial wave follows.

    python profiles/riccati_ab.py [--reps 3] [--workload quadrotor --workload quadrotor_calm] [--variant minb7=-DTO_FRAG_MINB=7]
    python profiles/riccati_ab.py --reps 1 --workload quadrotor_calm --batch 528 --batch 1056 --batch 2112 --batch 3168 --batch 4096"""
import argparse, json, os, subprocess, sys, tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "libtrajopt_b200.so")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def build_variant(name, flags, tmp):
    subprocess.run(["bash", os.path.join(ROOT, "profiles", "scripts", "build_variant.sh"), name, "riccati_frag.cu", flags],
                   check=True, env=dict(os.environ, VARIANT_DIR=tmp), stdout=subprocess.DEVNULL)
    return os.path.join(tmp, f"lib_{name}.so")


def bench(lib, workload, batch, dump):
    env = dict(os.environ, LIBTRAJOPT_B200=lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", workload,
           "--no-cpu-baseline", "--no-e2e", "--dump-outputs", dump]
    if batch:
        cmd += ["--batch", str(batch)]
    out = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    line = [l for l in out.stdout.splitlines() if l.startswith("{")]
    if out.returncode or not line:
        raise SystemExit(f"bench.py failed on {lib}:\n{out.stderr[-2000:]}")
    d = json.loads(line[-1])
    ph = d["roofline"]["phase_ms"]
    return dict(step=d["ms_per_step"], R=ph["backward"], F=ph["forward"], L=ph["ladder"], C1E1=ph["cost_expansion"] + ph["expand"],
                phases=ph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", action="append", default=[])
    ap.add_argument("--batch", type=int, action="append", default=[], help="batch sizes (default: the workload's)")
    ap.add_argument("--variant", action="append", default=[], metavar="NAME=FLAGS", help="riccati_frag.cu built with FLAGS")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    workloads = args.workload or ["quadrotor", "quadrotor_calm"]
    tmp = tempfile.mkdtemp(prefix="riccati_ab_")
    libs = {"default": DEFAULT}
    for kv in args.variant:
        name, flags = kv.split("=", 1)
        libs[f"{name} ({flags})"] = build_variant(name, flags, tmp)
    print(f"card: {card()}", flush=True)
    results, identical = [], True
    for wl in workloads:
        for batch in (args.batch or [0]):
            runs = {name: [] for name in libs}
            dumps = []
            for r in range(args.reps):
                for name, lib in libs.items():
                    d = os.path.join(tmp, f"dump_{wl}_{batch}_{len(dumps)}")
                    res = bench(lib, wl, batch, d)
                    runs[name].append(res); dumps.append((name, d))
                    print(f"  {wl} B={batch or 'default'}  {name:36s} step {res['step']:.4f}  R {res['R']:.4f}  F {res['F']:.4f}  "
                          f"L {res['L']:.4f}  C1+E1 {res['C1E1']:.4f}", flush=True)
            ref_name, ref = dumps[0]
            for name, d in dumps[1:]:
                for f in sorted(os.listdir(ref)):
                    a, b = np.load(os.path.join(ref, f)), np.load(os.path.join(d, f))
                    if a.shape != b.shape or not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
                        identical = False
                        print(f"  DUMP DIFFERS: {wl} {f} of {name} against {ref_name}")
            for name, rs in runs.items():
                rng = lambda k: f"{min(x[k] for x in rs):.3f}-{max(x[k] for x in rs):.3f}"
                print(f"{wl} B={batch or 'default'}  {name:36s} step {rng('step')}  R {rng('R')}  F {rng('F')}  L {rng('L')}  C1+E1 {rng('C1E1')}",
                      flush=True)
            results.append(dict(workload=wl, batch=batch, runs=runs))
    print(f"dumps bit-identical within every workload and batch: {identical}")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card(), results=results, identical=identical), fh, indent=1)
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()
