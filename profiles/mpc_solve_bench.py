"""Closed-loop MPC with a solve per step on the device (to_mpc_solve) against the same loop scripted on the host, and against to_mpc_run.

The BASELINE problem (error-state Quadrotor, B = 4096, N = 101, u in [0, 10] + Goal, record path), each instance tracking its own window of
the zig-zag reference of profiles/mpc_bench.py, T = 50 timed MPC steps after 2 untimed ones.  Arms, alternated in one call `--runs` times:
  solve_b{3,10,20}  mpc_setup, then mpc_solve(T, iterations=b) with Altro's default tolerances, timed to the synchronising mpc_history;
  scripted_b3       per step update_trajectory, solve(iterations=3), controls and merit (host reads), the plant on a second handle,
                    shift_trajectory(1), set_initial_state; set_penalties with the shared penalties first, as mpc_solve does;
  run_it3           mpc_run(T, 3): three plain iLQR iterations per step;
  loose_b{10,20}    mpc_solve with tolerances so loose that each instance stops at its first iteration that lowers the merit.
Reported per arm: ms per MPC step, kernel launches per step; for the solve arms the iterations used per step and instance (min, median, max),
the status counts, and the c_max of the applied plans (max over the finite values, median, how many were not finite).  For run_it3 the same
violation is read by a scripted replay of mpc_run's loop (to_max_violation after the iterations and the merit; the first run only, untimed).  Also: whether solve_b3 and scripted_b3 agree bit for bit (history and
statistics), (T(20) - T(10)) / 10 for the default and the loose tolerances with whether the iterations used at budget 20 stayed below 10
(then it is the cost of an idle iteration), and the card's name and power limit, read in the same run.
    python profiles/mpc_solve_bench.py [--T 50] [--runs 2] [--B 4096] [--out FILE]"""
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
from instance_weights_bench import card  # noqa: E402
from mpc_bench import WARM, launches, zigzag_reference  # noqa: E402

BUDGETS = (3, 10, 20)
STATS = ("status", "iterations", "iterations_outer", "c_max")


def _stats(h):
    return {f: getattr(h, f) for f in STATS}


# every instance stops after its first iteration that lowers the merit: the iterations after it, up to the budget, are idle
LOOSE = dict(cost_tolerance=1e9, cost_tolerance_intermediate=1e9, gradient_tolerance=1e9, gradient_tolerance_intermediate=1e9, constraint_tolerance=1e9)


def device_solve(B, T, budget, Xref, Uref, **opts):
    p = problems.quadrotor(B=B, error_state=True)
    TO.mpc_setup(p, WARM + T, Xref=Xref, Uref=Uref)
    TO.mpc_solve(p, WARM, iterations=budget, **opts)  # (creates the per-instance penalty table)
    TO.mpc_history(p)
    l0 = launches(p)
    t0 = time.perf_counter()
    TO.mpc_solve(p, T, iterations=budget, **opts)
    hist = TO.mpc_history(p)                          # synchronises
    ms = (time.perf_counter() - t0) * 1e3 / T
    out = (ms, (launches(p) - l0) / T, hist, _stats(TO.mpc_solve_history(p)))
    p.close()
    return out


def _plant(p):
    obj = TO.LQRObjective(np.ones(p.n), np.ones(p.m), np.ones(p.n), np.zeros(p.n), 2)
    return TO.Problem(p.model, obj, p.x0, float(p.spec.dt[0]), error_state=True)


def scripted(B, T, budget, Xref, Uref, solve=True):
    """the scripted loop: solve(iterations=budget) per step, or (solve=False) mpc_run's rollout + ilqr_step(budget) with the max violation
    of each applied plan read after the iterations"""
    p = problems.quadrotor(B=B, error_state=True)
    plant = _plant(p)
    if solve:
        for i in range(len(p.constraints)):
            TO.set_penalties(p, i, TO.penalty(p, i))
    X, U, J, S = [p.x0.copy()], [], [], {f: [] for f in STATS}

    def step(j):
        TO.update_trajectory(p, Xref, Uref, 1 + j)
        if solve:
            st = TO.solve(p, iterations=budget)
            for f in STATS:
                S[f].append(getattr(st, f).copy())
        else:
            TO.rollout(p)
            TO.ilqr_step(p, budget)
        u = TO.controls(p)[:, 0].copy()
        J.append(TO.merit(p).copy())
        if not solve:       # (after the merit: to_max_violation recomputes J from the trajectory, which the line search left)
            S["c_max"].append(TO.max_violation(p).copy())
        TO.set_initial_state(plant, p.x0)
        TO.initial_controls(plant, u[:, None, :])
        TO.rollout(plant)
        xn = TO.states(plant)[:, 1].copy()
        TO.shift_trajectory(p, 1)
        TO.set_initial_state(p, xn)
        X.append(xn); U.append(u)

    for j in range(WARM):
        step(j)
    l0 = launches(p, plant)
    t0 = time.perf_counter()
    for j in range(WARM, WARM + T):
        step(j)
    ms = (time.perf_counter() - t0) * 1e3 / T
    out = (ms, (launches(p, plant) - l0) / T, (np.stack(X, 1), np.stack(U, 1), np.stack(J, 1)),
           {f: np.stack(v, 1) for f, v in S.items() if v})
    p.close(); plant.close()
    return out


def device_run(B, T, iters, Xref, Uref):
    p = problems.quadrotor(B=B, error_state=True)
    TO.mpc_setup(p, WARM + T, Xref=Xref, Uref=Uref)
    TO.mpc_run(p, WARM, iters)
    TO.mpc_history(p)
    l0 = launches(p)
    t0 = time.perf_counter()
    TO.mpc_run(p, T, iters)
    hist = TO.mpc_history(p)
    ms = (time.perf_counter() - t0) * 1e3 / T
    out = (ms, (launches(p) - l0) / T, hist)
    p.close()
    return out


def summary(stats, timed_from=WARM):
    """iterations used and statuses of the timed steps, and the violation of the applied plans"""
    it = stats["iterations"][:, timed_from:]
    st = stats["status"][:, timed_from:]
    names, counts = np.unique([TO.SOLVE_STATUS_NAMES.get(int(s), str(int(s))) for s in st.ravel()], return_counts=True)
    per_step = lambda f: [int(f(it, axis=0).min()), int(f(it, axis=0).max())]
    return {"iterations_min": int(it.min()), "iterations_median": float(np.median(it)), "iterations_max": int(it.max()),
            "per_step_min_range": per_step(np.min), "per_step_max_range": per_step(np.max),
            "status_counts": dict(zip(names.tolist(), counts.tolist())), **violation(stats["c_max"][:, timed_from:])}


def violation(c):
    """the max violation of the applied plans over the finite values, their median, and how many (instance, step) plans were not finite"""
    fin = np.isfinite(c)
    return {"c_max_max_finite": float(c[fin].max()), "c_max_median": float(np.median(c[fin])), "c_max_nonfinite": int((~fin).sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=50); ap.add_argument("--runs", type=int, default=2); ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, T = a.B, a.T
    base = problems.quadrotor(B=B, error_state=True)
    Xref, Uref = zigzag_reference(base, WARM + T - 1 + base.N)
    base.close()
    res = {"card": card(), "B": B, "N": 101, "T": T, "runs": {}}
    log = lambda k, v: res["runs"].setdefault(k, []).append(v)
    for r in range(a.runs):
        dev = {}
        for b in BUDGETS:
            d = device_solve(B, T, b, Xref, Uref)
            dev[b] = d
            entry = {"ms_per_step": round(d[0], 3), "launches_per_step": d[1], **summary(d[3])}
            log(f"solve_b{b}", entry)
            print(f"solve budget={b} run={r}", entry, flush=True)
        s = scripted(B, T, 3, Xref, Uref)
        entry = {"ms_per_step": round(s[0], 3), "launches_per_step": s[1], **summary(s[3])}
        log("scripted_b3", entry)
        print(f"scripted budget=3 run={r}", entry, flush=True)
        d = device_run(B, T, 3, Xref, Uref)
        entry = {"ms_per_step": round(d[0], 3), "launches_per_step": d[1]}
        if r == 0:   # the violation of the applied plans, from an untimed replay of the same loop
            replay = scripted(B, T, 3, Xref, Uref, solve=False)
            entry.update(violation(replay[3]["c_max"][:, WARM:]))
            entry["replay_bit_identical"] = all(np.array_equal(x, y, equal_nan=True) for x, y in zip(d[2], replay[2]))
        log("run_it3", entry)
        print(f"mpc_run iterations=3 run={r}", entry, flush=True)
        same = all(np.array_equal(x, y, equal_nan=True) for x, y in zip(dev[3][2], s[2]))
        same = same and all(np.array_equal(dev[3][3][f], s[3][f], equal_nan=True) for f in STATS)
        log("bit_identical_b3", bool(same))
        print(f"run={r} device and scripted solve histories bit-identical: {same}", flush=True)
        idle = {}
        for b in (10, 20):   # the same step with loose tolerances: every instance stops early, the rest of the budget is idle
            idle[b] = device_solve(B, T, b, Xref, Uref, **LOOSE)
            entry = {"ms_per_step": round(idle[b][0], 3), "launches_per_step": idle[b][1], **summary(idle[b][3])}
            log(f"loose_b{b}", entry)
            print(f"loose tolerances budget={b} run={r}", entry, flush=True)
        for name, d10, d20 in (("default", dev[10], dev[20]), ("loose", idle[10], idle[20])):
            within = int(d20[3]["iterations"][:, WARM:].max()) < 10
            v = (d20[0] - d10[0]) / 10
            log(f"T20_minus_T10_over_10_{name}", {"ms": round(v, 4), "budget20_max_iterations_below_10": within})
            print(f"run={r} {name}: (T(20) - T(10)) / 10 = {v:.4f} ms (iterations used at budget 20 below 10: {within})", flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
