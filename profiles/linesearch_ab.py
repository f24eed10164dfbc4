#!/usr/bin/env python3
"""A/B of the line search's knot loop for the compact problem class on one GPU: the default library (rollout_compact) against the
variant built with -DTO_FWD_COMPACT=0 (rollout_fast for every fast-path problem), `bench.py --gpus 1 --steps 20 --warmup 3` three times
each, alternated, with the card's name and power limit; phase times F (forward = pass 1), L (ladder = late passes) and C1 + E1
(cost_expansion + expand) and the step time; the `--dump-outputs` of every run compared bitwise.

    python profiles/linesearch_ab.py [--reps 3] [--workload quadrotor] [--out results.json]"""
import argparse, json, os, subprocess, sys, tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "libtrajopt_b200.so")
VARIANT = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "variants", "lib_fwd_loop.so")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bench(lib, workload, dump):
    env = dict(os.environ, LIBTRAJOPT_B200=lib)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "3", "--workload", workload,
                          "--no-cpu-baseline", "--dump-outputs", dump], capture_output=True, text=True, env=env, cwd=ROOT)
    line = [l for l in out.stdout.splitlines() if l.startswith("{")]
    if out.returncode or not line:
        raise SystemExit(f"bench.py failed on {lib}:\n{out.stderr[-2000:]}")
    d = json.loads(line[-1])
    ph = d["roofline"]["phase_ms"]
    return dict(step=d["ms_per_step"], F=ph["forward"], L=ph["ladder"], C1E1=ph["cost_expansion"] + ph["expand"],
                E2C2=ph["late_expansion"], R=ph["backward"], phases=ph)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default="quadrotor")
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="further libraries to alternate with the two")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="linesearch_ab_")
    variant = VARIANT
    if not os.path.exists(variant):
        subprocess.run(["bash", os.path.join(ROOT, "profiles", "scripts", "build_variant.sh"), "fwd_loop", "forward.cu", "-DTO_FWD_COMPACT=0"],
                       check=True, env=dict(os.environ, VARIANT_DIR=tmp), stdout=subprocess.DEVNULL)
        variant = os.path.join(tmp, "lib_fwd_loop.so")
    print(f"card: {card()}  workload: {args.workload}", flush=True)
    libs = {"rollout_fast (-DTO_FWD_COMPACT=0)": variant, "rollout_compact (default)": DEFAULT}
    libs.update(dict(kv.split("=", 1) for kv in args.lib))
    runs = {name: [] for name in libs}
    dumps = []
    for r in range(args.reps):
        for name, lib in libs.items():
            d = os.path.join(tmp, f"dump_{len(dumps)}")
            res = bench(lib, args.workload, d)
            runs[name].append(res); dumps.append((name, d))
            print(f"  {name:36s} step {res['step']:.4f}  F {res['F']:.4f}  L {res['L']:.4f}  C1+E1 {res['C1E1']:.4f}  "
                  f"E2/C2 {res['E2C2']:.4f}  R {res['R']:.4f}", flush=True)
    ref_name, ref = dumps[0]
    identical = True
    for name, d in dumps[1:]:
        for f in sorted(os.listdir(ref)):
            a, b = np.load(os.path.join(ref, f)), np.load(os.path.join(d, f))
            if a.shape != b.shape or not np.array_equal(a.view(np.uint8), b.view(np.uint8)):
                identical = False
                print(f"  DUMP DIFFERS: {f} of {name} against {ref_name}")
    print(f"dumps bit-identical across all {len(dumps)} runs: {identical}")
    for name, rs in runs.items():
        rng = lambda k: f"{min(x[k] for x in rs):.3f}-{max(x[k] for x in rs):.3f}"
        print(f"{name:36s} step {rng('step')}  F {rng('F')}  L {rng('L')}  C1+E1 {rng('C1E1')}  E2/C2 {rng('E2C2')}  R {rng('R')}")
    fa, fb = runs["rollout_fast (-DTO_FWD_COMPACT=0)"], runs["rollout_compact (default)"]
    print(f"every default run faster than every variant run: {max(x['step'] for x in fb) < min(x['step'] for x in fa)}")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card(), runs=runs, identical=identical), fh, indent=1)
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()
