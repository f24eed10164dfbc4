"""Throughput of solve_queue with per-problem tables (to_solve_queue_tables) against chunked solve (one to_solve per chunk of B problems, the
chunk's rows set with the per-instance setters) over the same problems, arms alternated.

Workloads, the two uses the per-problem tables were added for:
- a horizon search: the constrained Cartpole swing-up (B = 1024 slots, N = 101, |u| <= 3 + Goal), M = 8 B problems with perturbed starts,
  each with one of 8 final times tf = 3.0, 3.5, ..., 6.5 (per-problem time steps);
- a limits and weights sweep: the BASELINE error-state Quadrotor (B = 4096 slots, N = 101, Goal + Bound), M = 8 B problems with perturbed
  starts, each with its own upper control limit (8, 9 or 10) and stage-cost weights (scaled by 1, 1.25, 1.5 or 1.75).
Default solve options.  Reported per arm: problems/s and the slot utilisation (instance-iterations run / (iterations x B), the iterations
counted from the handle's launch counters).  The per-problem results of the two arms are compared bit for bit.  The card's name and power
limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_weights_bench import card  # noqa: E402
from solve_queue_bench import _iterations_run  # noqa: E402

FIELDS = TO.SolveStats.FIELDS


def _cartpole(B):
    return problems.cartpole(B=B, u_bound=3.0, goal=True)


def _quadrotor(B):
    return problems.quadrotor(B=B, error_state=True)


def _horizons(p, M):
    return dict(dt=(3.0 + 0.5 * (np.arange(M) % 8)) / (p.N - 1))


def _limits_and_weights(p, M):
    bi = next(i for i, c in enumerate(p.constraints) if isinstance(c, TO.BoundConstraint))
    d = np.tile(TO.constraint_data(p, bi)[0], (M, 1))
    d[:, p.n:p.n + p.m] = (10.0 - np.arange(M) % 3)[:, None]                      # the upper control limits
    w = TO.cost_weights(p, 0)[0][None, :] * (1.0 + 0.25 * (np.arange(M) % 4))[:, None]
    return dict(constraint_data={bi: d}, cost_weights={0: w})


WORKLOADS = {"horizon_search": (_cartpole, 1024, _horizons), "limits_weights_sweep": (_quadrotor, 4096, _limits_and_weights)}


def _inputs(factory, tables, M):
    src = factory(M)
    x0, U0, kw = src.x0.copy(), TO.controls(src), tables(src, M)
    src.close()
    return x0, U0, kw


def queue(factory, B, x0, U0, kw):
    p = factory(B)
    _iterations_run(p)
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = TO.solve_queue(p, x0, U0, **kw)
    dt = time.perf_counter() - t
    its = _iterations_run(p)
    p.close()
    return dt, r, its


def chunked(factory, B, x0, U0, kw):
    M = x0.shape[0]
    p = factory(B)
    out = {f: [] for f in FIELDS}
    Xs, Us = [], []
    _iterations_run(p)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for c in range(0, M, B):
        idx = np.arange(c, c + B).clip(max=M - 1)
        if "dt" in kw:
            TO.set_time_steps(p, kw["dt"][idx])
        for j, rows in kw.get("cost_weights", {}).items():
            TO.set_cost_weights(p, j, rows[idx])
        for j, rows in kw.get("constraint_data", {}).items():
            TO.set_constraint_data(p, j, rows[idx])
        TO.set_initial_state(p, x0[idx])
        TO.initial_controls(p, U0[idx])
        for i in range(len(p.constraints)):   # each chunk starts as a fresh batch: lambda = 0, the initial penalties
            TO.set_multipliers(p, i, 0.0)
            TO.set_penalty(p, i, p._options.penalty_initial if getattr(p, "_options", None) else 1.0)
        st = TO.solve(p)
        k = min(B, M - c)
        for f in FIELDS:
            out[f].append(getattr(st, f)[:k])
        Xs.append(TO.states(p)[:k]); Us.append(TO.controls(p)[:k])
    dt = time.perf_counter() - t
    its = _iterations_run(p)
    p.close()
    return dt, {f: np.concatenate(v) for f, v in out.items()}, np.concatenate(Xs), np.concatenate(Us), its


def _rows(kw, sl):
    return {k: (v[sl] if isinstance(v, np.ndarray) else {j: r[sl] for j, r in v.items()}) for k, v in kw.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2); ap.add_argument("--chunks", type=int, default=8)
    ap.add_argument("--workloads", default="horizon_search,limits_weights_sweep")
    ap.add_argument("--scale", type=int, default=1, help="divide B by this (rehearsal)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        factory, B, tables = WORKLOADS[name]
        B //= a.scale
        M = a.chunks * B
        x0, U0, kw = _inputs(factory, tables, M)
        w = res["workloads"].setdefault(name, {"B": B, "M": M, "runs": []})
        queue(factory, B, x0[:B], U0[:B], _rows(kw, slice(0, B)))          # warm-up of every shape the timed runs use
        for r in range(a.runs):
            tq, rq, itq = queue(factory, B, x0, U0, kw)
            tc, rc, Xc, Uc, itc = chunked(factory, B, x0, U0, kw)
            work = int(rq.iterations.sum())
            same = all(np.array_equal(getattr(rq, f), rc[f]) for f in FIELDS) and np.array_equal(rq.X, Xc) and np.array_equal(rq.U, Uc)
            entry = {"queue_s": round(tq, 3), "queue_problems_per_s": round(M / tq, 1), "queue_iterations": itq,
                     "queue_utilisation": round(work / (itq * B), 4),
                     "max_iterations_of_a_problem": int(rq.iterations.max()),
                     "chunked_s": round(tc, 3), "chunked_problems_per_s": round(M / tc, 1), "chunked_iterations": itc,
                     "chunked_utilisation": round(int(rc["iterations"].sum()) / (itc * B), 4),
                     "instance_iterations": work, "speedup": round(tc / tq, 3), "bit_identical": bool(same)}
            w["runs"].append(entry)
            print(name, f"run={r}", entry, flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
