"""Cost of per-instance AL penalties, and what the per-instance outer step does to to_solve.

1. ms per iLQR iteration on the BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path), three arms alternated, `--runs`
   times each:
     shared          penalties shared by the batch (no per-instance tables: the INST = false kernels);
     goals           per-instance goals (every goal equal to the shared one): the INST = true kernels, the yardstick;
     equal_penalties every instance's penalties set to the shared ones: the same numbers through the INST = true kernels (trajectory and
                     merit checked bit for bit against `shared`).
2. to_solve, shared penalties against rows equal to them, alternated, on the same problem and on Cartpole 1024 x 101 (|u| <= 3 + goal).
   The results are identical (tests/test_gpu_instance_penalties.py), so the difference is the outer loop's scheduling: the shared solve
   waits for its slowest inner loop at every outer iteration, the per-instance one takes each instance's outer step on the device.
   Reports the wall time, the statuses, the iteration distribution and the batch iterations queued (line-search passes launched).
The card's name and power limit are read in the same run.
    python profiles/instance_penalties_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from trajopt_b200 import capi as K  # noqa: E402
from instance_goals_bench import time_steps  # noqa: E402
from instance_weights_bench import card  # noqa: E402


def equal_rows(p):
    for i in range(len(p.constraints)):
        TO.set_penalties(p, i, TO.penalty(p, i))
    return p


def solve_run(p):
    lib, h = p._lib, p._h
    pms = (C.c_double * K.PHASE_COUNT)(); pl = (C.c_int64 * K.PHASE_COUNT)()
    lib.to_get_phase_times(h, pms, pl, 1)                 # reset the counters
    K.check(lib, h, lib.to_synchronize(h))
    t = time.perf_counter()
    st = TO.solve(p)
    K.check(lib, h, lib.to_synchronize(h))
    wall = time.perf_counter() - t
    lib.to_get_phase_times(h, pms, pl, 1)
    its = np.asarray(st.iterations)
    # batch iterations queued: launches of the first line-search pass, one per iteration
    return st, {"wall_s": round(wall, 4), "batch_iterations": int(pl[K.PHASE_FORWARD]),
                "status": {TO.SOLVE_STATUS_NAMES[int(s)]: int(c) for s, c in zip(*np.unique(st.status, return_counts=True))},
                "iterations": {"mean": float(np.mean(its)), "min": int(its.min()), "p50": float(np.percentile(its, 50)),
                               "p90": float(np.percentile(its, 90)), "max": int(its.max())},
                "outer": {"min": int(np.min(st.iterations_outer)), "max": int(np.max(st.iterations_outer))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N

    def shared():
        return problems.quadrotor(B=B, N=N, error_state=True)

    def goals():
        p = shared()
        TO.set_goal_state(p, np.tile(p.xf, (B, 1)))
        return p

    arms = (("shared", shared), ("goals", goals), ("equal_penalties", lambda: equal_rows(shared())))
    res = {"card": card(), "B": B, "N": N, "runs": {k: [] for k, _ in arms}}
    for r in range(a.runs):
        dumps = {}
        for name, mk in arms:
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if name in ("shared", "equal_penalties"):
                dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["shared"], dumps["equal_penalties"]))
        res.setdefault("equal_penalties_bit_identical", []).append(bool(same))

    solves = {"quadrotor": shared, "cartpole": lambda: problems.cartpole(B=1024, N=101, u_bound=3.0, goal=True)}
    res["solve"] = {}
    for pname, mk in solves.items():
        out = {"shared": [], "equal_penalties": []}
        for r in range(a.runs):
            stats = {}
            for arm in ("shared", "equal_penalties"):
                p = mk() if arm == "shared" else equal_rows(mk())
                st, entry = solve_run(p)
                stats[arm] = (st, TO.states(p), TO.controls(p))
                out[arm].append(entry)
                p.close()
                print(pname, arm, r, entry, flush=True)
            (s0, X0, U0), (s1, X1, U1) = stats["shared"], stats["equal_penalties"]
            same = all(np.array_equal(getattr(s0, f), getattr(s1, f)) for f in TO.SolveStats.FIELDS)
            out.setdefault("identical", []).append(bool(same and np.array_equal(X0, X1) and np.array_equal(U0, U1)))
        res["solve"][pname] = out
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
