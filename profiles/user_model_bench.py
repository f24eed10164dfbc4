"""Per-iteration time of ilqr_step on user dynamics models of the padded size classes (8, 4) and (16, 8), against the built-in Quadrotor.

Workloads, B = 4096 instances, N = 101 knots, Goal + Bound, diagonal costs:
  * quadrotor_builtin : the built-in CUDA Quadrotor on the full-state path (n = 13, m = 4);
  * quadrotor_rec168  : a recorded copy of the same dynamics (AutodiffDynamics, 120 instructions), which runs as class (16, 8);
  * planar_rec84      : a recorded planar quadrotor (6, 2), which runs as class (8, 4).
Arms are alternated `--runs` times; each timed window is `--steps` iterations after `--warmup`, closed by a device synchronise.  Every
arm starts from hover controls, so the recorded and built-in Quadrotors compute the same iterations up to rounding.  The card's name and
power limit are read in the same run."""
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
from recorded_classes import planar_quadrotor_model, quadrotor_model  # noqa: E402


def _quadrotor(B, N, recorded):
    model = quadrotor_model() if recorded else TO.Quadrotor()
    ref = TO.problems.quadrotor(B=1, N=N, dt=0.05)
    obj = TO.LQRObjective(np.full(13, 1e-2), np.full(4, 1e-1), np.full(13, 10.0), ref.xf, N)
    cons = TO.ConstraintList(13, 4, N)
    TO.add_constraint(cons, TO.BoundConstraint(13, 4, u_min=0.2, u_max=6.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(ref.xf), N)
    x0 = np.tile(ref.x0[0], (B, 1))
    x0[:, :3] += 0.1 * np.random.default_rng(1).standard_normal((B, 3))
    p = TO.Problem(model, obj, x0, float(TO.gettimes(ref)[-1]), xf=ref.xf, constraints=cons, dt=0.05)
    ref.close()
    U = np.tile(TO.Quadrotor().hover_control(), (B, N - 1, 1))
    TO.initial_controls(p, np.concatenate([U, np.zeros((B, N - 1, p.m - 4))], axis=-1) if recorded else U)
    return p


def _planar(B, N):
    xf = np.array([1.0, 0.5, 0.0, 0.0, 0.0, 0.0])
    obj = TO.LQRObjective(np.full(6, 0.1), np.full(2, 0.01), np.full(6, 50.0), xf, N)
    cons = TO.ConstraintList(6, 2, N)
    TO.add_constraint(cons, TO.BoundConstraint(6, 2, u_min=0.0, u_max=12.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    x0 = 0.1 * np.random.default_rng(2).standard_normal((B, 6))
    p = TO.Problem(planar_quadrotor_model(), obj, x0, 0.05 * (N - 1), xf=xf, constraints=cons)
    TO.initial_controls(p, np.tile([4.905, 4.905, 0.0, 0.0], (B, N - 1, 1)))
    return p


ARMS = {"quadrotor_builtin": lambda B, N: _quadrotor(B, N, False), "quadrotor_rec168": lambda B, N: _quadrotor(B, N, True),
        "planar_rec84": _planar}


def time_arm(name, B, N, steps, warmup):
    p = ARMS[name](B, N)
    TO.rollout(p)
    TO.ilqr_step(p, warmup)
    torch.cuda.synchronize()
    t = time.perf_counter()
    TO.ilqr_step(p, steps)
    assert p._lib.to_synchronize(p._h) == 0
    ms = (time.perf_counter() - t) * 1e3 / steps
    out = dict(ms_per_iteration=ms, n=p.n, m=p.m, backward=TO.kernel_choice(p)["backward"], linesearch=TO.kernel_choice(p)["linesearch"],
               merit_finite=bool(np.all(np.isfinite(TO.merit(p)))))
    p.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("user_model_bench: no CUDA device")
    res = {"card": card(), "B": a.B, "N": a.N, "steps": a.steps, "runs": []}
    for r in range(a.runs):
        res["runs"].append({name: time_arm(name, a.B, a.N, a.steps, a.warmup) for name in ARMS})
        print(json.dumps(res["runs"][-1]), flush=True)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
