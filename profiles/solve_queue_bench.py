"""Throughput of solve_queue (M problems through B slots, refilled on the device) against chunked solve (one to_solve per chunk of B problems)
over the same problems, arms alternated.

Workloads: the BASELINE error-state Quadrotor (B = 4096 slots, N = 101, Goal + Bound, default solve options) with M = 8 B problems whose
starts and goals are perturbed, and the constrained Cartpole swing-up (B = 1024 slots, N = 101, |u| <= 3 + Goal) with M = 8 B perturbed starts
and goals.  Reported per arm: problems/s and the slot utilisation (instance-iterations
run / (iterations x B), the iterations counted from the handle's launch counters).  The per-problem results of the two arms
are compared bit for bit.  The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import _capi as K  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_weights_bench import card  # noqa: E402

FIELDS = TO.SolveStats.FIELDS


def _quadrotor(B):
    return problems.quadrotor(B=B, error_state=True)


def _cartpole(B):
    return problems.cartpole(B=B, u_bound=3.0, goal=True)


WORKLOADS = {"quadrotor": (_quadrotor, 4096), "cartpole": (_cartpole, 1024)}


def _inputs(factory, M, seed=5):
    src = factory(M)
    x0, U0 = src.x0.copy(), TO.controls(src)
    xf = np.tile(np.asarray(src.xf, dtype=float), (M, 1))
    k = 3 if src.n == 13 else 2
    xf[:, :k] += 0.2 * np.random.default_rng(seed).uniform(-1, 1, (M, k))
    src.close()
    return x0, U0, xf


def _iterations_run(p):
    """iterations enqueued since the last call (each iteration launches one dynamics expansion on the main stream), counters reset"""
    ms, n = (C.c_double * K.PHASE_COUNT)(), (C.c_int64 * K.PHASE_COUNT)()
    p._lib.to_get_phase_times(p._h, ms, n, 1)
    return int(n[K.PHASE_EXPAND])


def queue(factory, B, x0, U0, xf):
    p = factory(B)
    _iterations_run(p)
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = TO.solve_queue(p, x0, U0, xf=xf)
    dt = time.perf_counter() - t
    its = _iterations_run(p)
    p.close()
    return dt, r, its


def chunked(factory, B, x0, U0, xf):
    M = x0.shape[0]
    p = factory(B)
    out = {f: [] for f in FIELDS}
    Xs, Us = [], []
    _iterations_run(p)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for c in range(0, M, B):
        idx = np.arange(c, c + B).clip(max=M - 1)
        TO.set_initial_state(p, x0[idx])
        TO.initial_controls(p, U0[idx])
        TO.set_goal_state(p, xf[idx])
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2); ap.add_argument("--chunks", type=int, default=8)
    ap.add_argument("--workloads", default="quadrotor,cartpole"); ap.add_argument("--scale", type=int, default=1, help="divide B by this (rehearsal)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workloads": {}}
    for name in a.workloads.split(","):
        factory, B = WORKLOADS[name]
        B //= a.scale
        M = a.chunks * B
        x0, U0, xf = _inputs(factory, M)
        w = res["workloads"].setdefault(name, {"B": B, "M": M, "runs": []})
        queue(factory, B, x0[:B], U0[:B], xf[:B])          # warm-up of every shape the timed runs use
        for r in range(a.runs):
            tq, rq, itq = queue(factory, B, x0, U0, xf)
            tc, rc, Xc, Uc, itc = chunked(factory, B, x0, U0, xf)
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
