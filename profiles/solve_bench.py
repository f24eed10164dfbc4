"""Solve-to-convergence measurement (to_solve, DESIGN.md 5d).  Two workloads, default solve options:
  * the BASELINE Quadrotor (4096 x 101, error state, Goal + Bound; problems.quadrotor);
  * the notebook Cartpole with |u| <= 3 + goal, B = 1024, perturbed x0 (problems.cartpole).
For each: wall time of the solve (device-synchronised), problems solved per second, the histogram of per-instance iterations, the
instance-iterations executed against B x (max iterations) -- what a loop without retirement executes -- and the time of one iteration with
100 / 50 / 10 / 1 % of the instances ACTIVE (step_time).
Prints the card name and power limit of the run.  Usage: python profiles/solve_bench.py [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402

P = TO.problems


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().split("\n")[0]
        return out
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def solve_timed(build):
    p = build()
    p._call("to_synchronize")
    t0 = time.perf_counter()
    st = TO.solve(p)
    p._call("to_synchronize")
    return time.perf_counter() - t0, st, p


def step_time(build, frac, K=20, reps=3):
    """ms per iteration with a fraction `frac` of the instances ACTIVE.  The first B * frac instances start from the problem's initial guess;
    the others are copies (x0, controls, multipliers) of instances that a first solve brought to SOLVE_SUCCEEDED.  Started at a solution, a copy
    ends its inner loop in its first iteration and is retired: it waits, running no kernel, until the ACTIVE instances reach the iteration
    cap, and the outer step then finds it within constraint_tolerance (1e-2 here).  The time of one iteration is
    (T(1 + K) - T(1)) / K, T(c) = wall time of a solve capped at c iterations: the first iteration, in which every instance is ACTIVE, and
    the solve's fixed costs cancel.  Returns the time and the instance-iterations the ACTIVE / retired instances ran in iterations 2..1+K."""
    warm = build()
    sw = TO.solve(warm)
    ok = np.nonzero(sw.status == TO.capi.SOLVE_SUCCEEDED)[0]
    Xw, Uw = warm.x0.copy(), TO.controls(warm)
    lw = [TO.multipliers(warm, c) for c in warm.constraints.constraints]
    warm.close()
    B = len(sw.status)
    n_act = max(1, int(round(B * frac)))
    src = ok[np.arange(B - n_act) % len(ok)]

    def timed(cap):
        p = build()
        x0 = p.x0.copy(); x0[n_act:] = Xw[src]
        TO.set_initial_state(p, x0)
        U = TO.controls(p).copy(); U[n_act:] = Uw[src]
        TO.initial_controls(p, U)
        for c, l in zip(p.constraints.constraints, lw):
            lam = TO.multipliers(p, c)
            lam[n_act:] = l[src]
            TO.set_multipliers(p, c, lam)
        p._call("to_synchronize")
        t0 = time.perf_counter()
        st = TO.solve(p, iterations=cap, constraint_tolerance=1e-2)
        p._call("to_synchronize")
        dt = time.perf_counter() - t0
        p.close()
        return dt, st

    t1 = min(timed(1)[0] for _ in range(reps))
    runs = [timed(1 + K) for _ in range(reps)]
    tk = min(r[0] for r in runs)
    st = runs[0][1]
    return {"ms_per_iteration": round((tk - t1) / K * 1e3, 4), "active_instance_iterations": int(st.iterations[:n_act].sum() - n_act),
            "retired_instance_iterations": int(st.iterations[n_act:].sum() - (B - n_act))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    res = {"card": card()}
    loads = {
        "quadrotor_4096x101": lambda: P.quadrotor(B=4096, N=101, error_state=True),
        "cartpole_1024x101": lambda: P.cartpole(B=1024, N=101, u_bound=3.0, goal=True),
    }
    for name, build in loads.items():
        solve_timed(build)                   # warm-up (module load, first launches)
        times, st = [], None
        for _ in range(args.reps):
            dt, st, p = solve_timed(build)
            times.append(dt)
            p.close()
        it = st.iterations
        hist, edges = np.histogram(it, bins=[0, 10, 20, 30, 40, 60, 80, 100, 150, 200, 301])
        names, counts = np.unique(st.status_names(), return_counts=True)
        r = {"B": int(len(it)), "solve_s": [round(t, 4) for t in times], "solved_per_s": round(len(it) / float(np.median(times)), 1),
             "status": dict(zip(names.tolist(), counts.tolist())),
             "iterations_min_median_max": [int(it.min()), float(np.median(it)), int(it.max())],
             "iteration_histogram": {f"{int(a)}-{int(b) - 1}": int(c) for a, b, c in zip(edges[:-1], edges[1:], hist)},
             "instance_iterations_executed": int(it.sum()), "instance_iterations_without_retirement": int(len(it) * it.max())}
        r["step_at_active_fraction"] = {str(f): step_time(build, f) for f in (1.0, 0.5, 0.1, 0.01)}
        res[name] = r
        print(name, json.dumps(r), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
