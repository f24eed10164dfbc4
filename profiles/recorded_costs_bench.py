"""Per-iteration time of ilqr_step on user dynamics models with each kind of cost, at the padded size classes (8, 4) and (16, 8).

Workloads, B = 4096 instances, N = 101 knots, Bound + Goal constraints:
  * planar_*: the planar quadrotor (6, 2), class (8, 4);
  * arm_*:    the 7-joint arm (14, 7), class (16, 8);
each with a DiagonalCost (LQRObjective), a dense QuadraticCost (every entry of Q, R and H nonzero) and an AutodiffCost restating the
DiagonalCost.  The first two run the in-kernel expansion of k_riccati; the user cost runs the materialised expansion (k_al_expansion,
k_error_expansion) and k_riccati_dense.  Arms are alternated `--runs` times; each timed window is `--steps` iterations after `--warmup`,
closed by a device synchronise.  The card's name and power limit are read in the same run.  The bytes of the materialised expansion
EH = B N (n + m)^2 8 are computed from the shapes."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import trajopt_b200 as TO  # noqa: E402
from instance_weights_bench import card  # noqa: E402
from recorded_classes import arm7_model, planar_quadrotor_model  # noqa: E402
from recorded_costs import HOVER, dense_cost, diagonal_as_user_cost  # noqa: E402

MODELS = {"planar": (planar_quadrotor_model, np.array([1.0, 0.5, 0.0, 0.0, 0.0, 0.0]), (0.0, 12.0), HOVER),
          "arm": (arm7_model, np.concatenate([np.full(7, 0.5), np.zeros(7)]), (-4.0, 4.0), 0.0)}


def _problem(model_name, cost, B, N):
    make, xf, (ulo, uhi), u0 = MODELS[model_name]
    model = make()
    n, m = model.n, model.m
    Qd, Rd, Qf = np.full(n, 0.1), np.full(m, 0.01), np.full(n, 50.0)
    if cost == "diagonal":
        obj = TO.LQRObjective(Qd, Rd, Qf, xf, N)
    elif cost == "dense":
        obj = TO.Objective([dense_cost(n, m, 1)] * (N - 1) + [dense_cost(n, m, 2, terminal=True)])
    else:
        obj = TO.Objective([diagonal_as_user_cost(Qd, Rd, xf)] * (N - 1) + [diagonal_as_user_cost(Qf, Rd, xf, terminal=True)])
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=ulo, u_max=uhi), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    x0 = 0.1 * np.random.default_rng(2).standard_normal((B, n))
    p = TO.Problem(model, obj, x0, 0.02 * (N - 1), xf=xf, constraints=cons)
    U = np.zeros((B, N - 1, p.m))
    U[..., :m] = u0
    TO.initial_controls(p, U)
    return p


ARMS = [(mdl, c) for mdl in MODELS for c in ("diagonal", "dense", "user")]


def time_arm(model_name, cost, B, N, steps, warmup):
    p = _problem(model_name, cost, B, N)
    TO.rollout(p)
    TO.ilqr_step(p, warmup)
    torch.cuda.synchronize()
    t = time.perf_counter()
    TO.ilqr_step(p, steps)
    assert p._lib.to_synchronize(p._h) == 0
    ms = (time.perf_counter() - t) * 1e3 / steps
    choice = TO.kernel_choice(p)
    out = dict(ms_per_iteration=ms, n=p.n, m=p.m, backward=choice["backward"], linesearch=choice["linesearch"],
               merit_finite=bool(np.all(np.isfinite(TO.merit(p)))),
               EH_bytes=B * N * (p.n + p.m) ** 2 * 8 if choice["backward"] == "dense_dfma" else 0)
    p.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=2); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("recorded_costs_bench: no CUDA device")
    res = {"card": card(), "B": a.B, "N": a.N, "steps": a.steps, "runs": []}
    for r in range(a.runs):
        res["runs"].append({f"{mdl}_{c}": time_arm(mdl, c, a.B, a.N, a.steps, a.warmup) for mdl, c in ARMS})
        print(json.dumps(res["runs"][-1]), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
