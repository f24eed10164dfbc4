"""Cost of the integration rule (to_set_integration).

ms per iLQR iteration and the phase times (to_get_phase_times: expansion E, forward pass F, ...) on the BASELINE problem (error-state
Quadrotor, B = 4096, N = 101, record path), five arms alternated, `--runs` times each:
  default   a handle that never called the setter (RK4);
  RK4       RK4 set explicitly (trajectory and merit checked bit for bit against `default`);
  RK3, RK2, Euler.
The card's name and power limit are read in the same run.
    python profiles/integration_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
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
from instance_weights_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N

    def arm(rule):
        def make():
            p = problems.quadrotor(B=B, N=N, error_state=True)
            if rule is not None:
                TO.set_integration(p, rule)
            return p
        return make

    arms = (("default", arm(None)), ("RK4", arm("RK4")), ("RK3", arm("RK3")), ("RK2", arm("RK2")), ("Euler", arm("Euler")))
    res = {"card": card(), "B": B, "N": N, "runs": {k: [] for k, _ in arms}}
    for r in range(a.runs):
        dumps = {}
        for name, mk in arms:
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if name in ("default", "RK4"):
                dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["default"], dumps["RK4"]))
        res.setdefault("rk4_bit_identical", []).append(bool(same))
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
