"""Cost of per-instance constraint data.

BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path), four arms, alternated, `--runs` times each:
  shared       the control box shared by the batch (no per-instance tables: the INST = false kernels);
  goals        per-instance goals (to_set_goal_states, every goal equal to the shared one): the INST = true kernels, the yardstick;
  equal_boxes  every instance's control box set to the shared one: the same numbers through the INST = true kernels (the arm's trajectory
               and merit are checked bit for bit against `shared`);
  boxes        u_max drawn in [8, 12] per instance.
Obstacle workload (2-D DoubleIntegrator, B = 4096, N = 101, generic line search), alternated the same way:
  obstacles_shared  4 Circle obstacles shared by the batch;
  obstacles         4 Circle obstacles at random positions per instance.
Reports ms per iLQR iteration (to_ilqr_step, synchronised wall time) with the per-phase CUDA-event timers, then one to_solve of each
randomised arm: wall time, statuses and the iteration distribution.
    python profiles/instance_constraints_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
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


def obstacle_problem(B, N, rng=None):
    """2-D DoubleIntegrator from (0, 0) to (0, 4) among 4 Circle obstacles (shared, or at random positions per instance with rng)"""
    n, m = 4, 2
    xf = np.array([0.0, 4.0, 0, 0])
    obj = TO.LQRObjective(np.eye(n), 0.1 * np.eye(m), np.eye(n) * (N - 1), xf, N)
    cons = TO.ConstraintList(n, m, N)
    circ = TO.CircleConstraint(n, [0.3, -0.4, 0.2, -0.1], [1.0, 1.8, 2.6, 3.3], [0.3, 0.3, 0.3, 0.3])
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    TO.add_constraint(cons, circ, (2, N - 1))
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=-10, u_max=10), (1, N - 1))
    p = TO.Problem(TO.DoubleIntegrator(2), obj, np.zeros((B, n)), 4.0, xf=xf, constraints=cons)
    TO.initial_controls(p, 0.01 * np.random.default_rng(1).standard_normal((B, N - 1, m)))
    if rng is not None:
        rows = np.concatenate([rng.uniform(-0.6, 0.6, (B, 4)), rng.uniform(0.6, 3.4, (B, 4)), rng.uniform(0.2, 0.35, (B, 4))], axis=1)
        TO.set_constraint_data(p, circ, rows)
    return p


def solve_stats(p):
    t = time.perf_counter()
    st = TO.solve(p)
    its = np.asarray(st.iterations)
    return {"wall_s": round(time.perf_counter() - t, 3),
            "status": {TO.SOLVE_STATUS_NAMES[int(s)]: int(c) for s, c in zip(*np.unique(st.status, return_counts=True))},
            "iterations": {"mean": float(np.mean(its)), "min": int(its.min()), "p50": float(np.percentile(its, 50)),
                           "p90": float(np.percentile(its, 90)), "max": int(its.max())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N

    def box_index(p):
        return next(j for j, c in enumerate(p.constraints.constraints) if isinstance(c, TO.BoundConstraint))

    def shared():
        return problems.quadrotor(B=B, N=N, error_state=True)

    def goals():
        p = shared()
        TO.set_goal_state(p, np.tile(p.xf, (B, 1)))
        return p

    def equal_boxes():
        p = shared()
        j = box_index(p)
        TO.set_constraint_data(p, j, [p.constraints[j]] * B)
        return p

    def boxes():
        p = shared()
        j = box_index(p)
        rows = TO.constraint_data(p, j)
        nm = rows.shape[1] // 2
        rows[:, p.n:nm] = np.random.default_rng(5).uniform(8.0, 12.0, (B, p.m))
        TO.set_constraint_data(p, j, rows)
        return p

    arms = (("shared", shared), ("goals", goals), ("equal_boxes", equal_boxes), ("boxes", boxes),
            ("obstacles_shared", lambda: obstacle_problem(B, N)), ("obstacles", lambda: obstacle_problem(B, N, np.random.default_rng(7))))
    res = {"device": None, "B": B, "N": N, "runs": {k: [] for k, _ in arms}}
    try:
        import torch
        res["device"] = torch.cuda.get_device_name(0)
    except Exception:
        pass
    for r in range(a.runs):
        dumps = {}
        for name, mk in arms:
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if name in ("shared", "equal_boxes"):
                dumps[name] = (TO.states(p), TO.controls(p), TO.merit(p))
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
        same = all(np.array_equal(x, y) for x, y in zip(dumps["shared"], dumps["equal_boxes"]))
        res.setdefault("equal_boxes_bit_identical", []).append(bool(same))
    for name, mk in (("boxes", boxes), ("obstacles", arms[-1][1])):
        p = mk()
        res[f"solve_{name}"] = solve_stats(p)
        p.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
