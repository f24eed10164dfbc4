"""Cost of per-instance goals on the BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path).

Three arms, alternated, `--runs` times each: a shared goal, per-instance goals (LQRObjective: 2 costs, ~1 MB of linear terms) and per-instance
tracking references (TrackingObjective: N costs, ~56 MB).  Reports ms per iLQR iteration (to_ilqr_step, synchronised wall time) with the
per-phase CUDA-event timers, then to_solve wall time and statuses with per-instance goals drawn around the BASELINE goal.
    python profiles/instance_goals_bench.py [--steps 20] [--warmup 3] [--runs 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import _capi as K, problems  # noqa: E402

PHASES = (("expand", K.PHASE_EXPAND), ("cost_expansion", K.PHASE_COSTEXP), ("backward", K.PHASE_BACKWARD), ("forward", K.PHASE_FORWARD),
          ("ladder", K.PHASE_LADDER), ("late_expansion", K.PHASE_LATE))


def tracking_quadrotor(B, N, seed=1):
    base = problems.quadrotor(B=B, N=N, error_state=True, seed=seed)
    n, m = base.n, base.m
    uf = TO.Quadrotor().hover_control()
    Xref = np.linspace(base.x0[0], base.xf, N); Xref[:, 3:7] = base.xf[3:7]
    Uref = np.tile(uf, (N - 1, 1))
    obj = TO.TrackingObjective(np.full(n, 0.1), np.full(m, 0.01), Xref, Uref, Qf=np.full(n, 100.0))
    p = TO.Problem(TO.Quadrotor(), obj, base.x0, 5.0, xf=base.xf, constraints=base.constraints, error_state=True)
    TO.initial_controls(p, TO.controls(base))
    base.close()
    return p, Xref, Uref


def time_steps(p, steps, warmup):
    lib, h = p._lib, p._h
    TO.rollout(p)
    TO.ilqr_step(p, warmup); TO.merit(p)
    lib.to_set_phase_timing(h, 1)
    pms = (C.c_double * K.PHASE_COUNT)(); pl = (C.c_int64 * K.PHASE_COUNT)()
    lib.to_get_phase_times(h, pms, pl, 1)
    t = time.perf_counter()
    TO.ilqr_step(p, steps)
    K.check(lib, h, lib.to_synchronize(h))
    ms = (time.perf_counter() - t) * 1e3 / steps
    lib.to_get_phase_times(h, pms, pl, 1)
    lib.to_set_phase_timing(h, 0)
    return ms, {name: round(pms[i] / max(1, pl[i]), 4) for name, i in PHASES}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3); ap.add_argument("--B", type=int, default=4096); ap.add_argument("--N", type=int, default=101)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.B, a.N
    rng = np.random.default_rng(5)

    def shared():
        return problems.quadrotor(B=B, N=N, error_state=True)

    def goals():
        p = problems.quadrotor(B=B, N=N, error_state=True)
        xf = np.tile(p.xf, (B, 1)); xf[:, :3] += rng.uniform(-0.5, 0.5, (B, 3))
        TO.set_goal_state(p, xf)
        return p

    def tracking():
        p, Xref, Uref = tracking_quadrotor(B, N)
        Xb = np.tile(Xref, (B, 1, 1)); Xb[:, :, :3] += rng.uniform(-0.5, 0.5, (B, 1, 3))
        Ub = np.tile(np.vstack([Uref, Uref[-1:]]), (B, 1, 1))
        t = time.perf_counter(); TO.update_trajectory(p, Xb, Ub, 1); p._update_ms = (time.perf_counter() - t) * 1e3
        return p

    res = {"device": None, "B": B, "N": N, "runs": {k: [] for k in ("shared", "instance_goals", "instance_tracking")}}
    try:
        import torch
        res["device"] = torch.cuda.get_device_name(0)
    except Exception:
        pass
    for r in range(a.runs):
        for name, mk in (("shared", shared), ("instance_goals", goals), ("instance_tracking", tracking)):
            p = mk()
            ms, ph = time_steps(p, a.steps, a.warmup)
            entry = {"ms_per_step": round(ms, 4), "phase_ms": ph}
            if hasattr(p, "_update_ms"):
                entry["update_trajectories_ms"] = round(p._update_ms, 2)
            res["runs"][name].append(entry)
            p.close()
            print(name, r, entry, flush=True)
    p = goals()
    t = time.perf_counter()
    st = TO.solve(p)
    res["solve_instance_goals"] = {"wall_s": round(time.perf_counter() - t, 3),
                                   "status": {TO.SOLVE_STATUS_NAMES[int(s)]: int(c) for s, c in zip(*np.unique(st.status, return_counts=True))},
                                   "iterations_mean": float(np.mean(st.iterations))}
    p.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
