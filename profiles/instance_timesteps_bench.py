"""Cost of per-instance time steps (to_set_time_steps).

ms per iLQR iteration on the BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path), four arms alternated, `--runs` times
each:
  shared        one grid for the batch (no per-instance tables: the INST = false kernels);
  params        per-instance model parameters equal to the shared ones: the yardstick, the same INST = true dynamics and line-search kernels;
  equal_steps   every instance's time steps set to the shared grid: the same numbers through the INST = true kernels (trajectory and merit
                checked bit for bit against `shared`);
  drawn         tf_b drawn in [4, 6] s, uniform steps tf_b / (N - 1) per instance.
Then to_solve on the drawn arm: statuses and iteration statistics.  The card's name and power limit are read in the same run.
    python profiles/instance_timesteps_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_goals_bench import time_steps  # noqa: E402
from instance_penalties_bench import solve_run  # noqa: E402
from instance_weights_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N
    tf = np.random.default_rng(7).uniform(4.0, 6.0, B)

    def shared():
        return problems.quadrotor(B=B, N=N, error_state=True)

    def params():
        p = shared()
        TO.set_model_params(p, [p.model] * B)
        return p

    def equal_steps():
        p = shared()
        TO.set_time_steps(p, np.tile(p.spec.dt, (B, 1)))
        return p

    def drawn():
        p = shared()
        TO.set_time_steps(p, tf / (N - 1))
        return p

    arms = (("shared", shared), ("params", params), ("equal_steps", equal_steps), ("drawn", drawn))
    res = {"card": card(), "B": B, "N": N, "tf_range": [float(tf.min()), float(tf.max())], "runs": {k: [] for k, _ in arms}}
    for r in range(a.runs):
        dumps = {}
        for name, mk in arms:
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if name in ("shared", "equal_steps"):
                dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["shared"], dumps["equal_steps"]))
        res.setdefault("equal_steps_bit_identical", []).append(bool(same))

    p = drawn()
    st, entry = solve_run(p)
    p.close()
    res["solve_drawn"] = entry
    print("solve drawn", entry, flush=True)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
