"""Cost of per-instance model parameters on the BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path).

Three arms, alternated, `--runs` times each:
  shared       the model's parameters, shared by the batch (no per-instance rows: the INST = false kernels);
  equal_rows   every row set to the shared parameters: the same numbers through the INST = true kernels, so the difference to `shared`
               is the cost of reading the rows (the arm's trajectory and merit are checked bit for bit against `shared`);
  randomised   mass and J1..J3 drawn within +-20 % per instance, each instance starting from its own hover thrust.
Reports ms per iLQR iteration (to_ilqr_step, synchronised wall time) with the per-phase CUDA-event timers, then to_solve of the randomised
arm: wall time, statuses and the iteration distribution.
    python profiles/instance_params_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_goals_bench import time_steps  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N
    rng = np.random.default_rng(5)
    base = np.array(TO.Quadrotor().params)
    rows = np.tile(base, (B, 1)); rows[:, :4] *= 1.0 + rng.uniform(-0.2, 0.2, (B, 4))

    def shared():
        return problems.quadrotor(B=B, N=N, error_state=True)

    def equal_rows():
        p = problems.quadrotor(B=B, N=N, error_state=True)
        TO.set_model_params(p, np.tile(base, (B, 1)))
        return p

    def randomised():
        p = problems.quadrotor(B=B, N=N, error_state=True)
        TO.set_model_params(p, rows)
        hover0 = TO.Quadrotor().hover_control()
        hover = -rows[:, 6:7] * rows[:, 0:1] / 4.0                            # -g_z mass / 4 of each instance
        TO.initial_controls(p, TO.controls(p) - hover0[None, None, :] + hover[:, None, :])
        return p

    res = {"device": None, "B": B, "N": N, "runs": {k: [] for k in ("shared", "equal_rows", "randomised")}}
    try:
        import torch
        res["device"] = torch.cuda.get_device_name(0)
    except Exception:
        pass
    for r in range(a.runs):
        dumps = {}
        for name, mk in (("shared", shared), ("equal_rows", equal_rows), ("randomised", randomised)):
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["shared"], dumps["equal_rows"]))
        res.setdefault("equal_rows_bit_identical", []).append(bool(same))
    p = randomised()
    t = time.perf_counter()
    st = TO.solve(p)
    its = np.asarray(st.iterations)
    res["solve_randomised"] = {"wall_s": round(time.perf_counter() - t, 3),
                               "status": {TO.SOLVE_STATUS_NAMES[int(s)]: int(c) for s, c in zip(*np.unique(st.status, return_counts=True))},
                               "iterations": {"mean": float(np.mean(its)), "min": int(its.min()), "p50": float(np.percentile(its, 50)),
                                              "p90": float(np.percentile(its, 90)), "max": int(its.max())}}
    p.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
