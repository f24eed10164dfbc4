"""Cost of per-instance cost weights.

BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path), four arms, alternated, `--runs` times each:
  shared          the objective shared by the batch (no per-instance tables: the INST = false kernels);
  goals           per-instance goals (to_set_goal_states, every goal equal to the shared one): the INST = true kernels, the yardstick;
  equal_weights   every instance's weights set to the shared ones: the same numbers through the INST = true kernels (the arm's trajectory
                  and merit are checked bit for bit against `shared`);
  weights         Q and R of every cost scaled per instance by factors drawn in [0.5, 2].
Reports ms per iLQR iteration (to_ilqr_step, synchronised wall time) with the per-phase CUDA-event timers, then one to_solve of the
`weights` arm: wall time, statuses and the iteration distribution.  The card's name and power limit are read in the same run.
    python profiles/instance_weights_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_goals_bench import time_steps  # noqa: E402
from instance_constraints_bench import solve_stats  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return None


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

    def equal_weights():
        p = shared()
        for j, c in enumerate(p._cost_objs):
            TO.set_cost_weights(p, j, np.tile(TO.api._cost_weight_row(c), (B, 1)))
        return p

    def weights():
        p = shared()
        rng = np.random.default_rng(5)
        for j in range(len(p._cost_objs)):
            rows = TO.cost_weights(p, j)
            rows[:, :p.n + p.m] *= rng.uniform(0.5, 2.0, (B, p.n + p.m))   # DiagonalCost rows: Qd | Rd | c
            TO.set_cost_weights(p, j, rows)
        return p

    arms = (("shared", shared), ("goals", goals), ("equal_weights", equal_weights), ("weights", weights))
    res = {"card": card(), "B": B, "N": N, "runs": {k: [] for k, _ in arms}}
    for r in range(a.runs):
        dumps = {}
        for name, mk in arms:
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if name in ("shared", "equal_weights"):
                dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["shared"], dumps["equal_weights"]))
        res.setdefault("equal_weights_bit_identical", []).append(bool(same))
    p = weights()
    res["solve_weights"] = solve_stats(p)
    p.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
