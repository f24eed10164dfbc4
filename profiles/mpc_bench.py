"""Closed-loop MPC on the device (to_mpc_run) against the same loop scripted on the host through the existing entry points.

The BASELINE problem (error-state Quadrotor, B = 4096, N = 101, record path), each instance tracking its own window of a long reference along
the zig-zag of examples/Quadrotor.ipynb (the waypoints of problems.quadrotor_zigzag, offset per instance), T = 50 MPC steps of `iterations`
iLQR iterations each, iterations in {1, 3}.  The two loops run in the same call, alternated, `--runs` times:
  device    mpc_setup once, then one mpc_run(T, iterations), timed to the synchronising mpc_history;
  scripted  per step update_trajectory (per instance, from the host), rollout, ilqr_step, controls and merit (host reads), the plant on a
            second handle (N = 2: set_initial_state, initial_controls, rollout, states), shift_trajectory(1), set_initial_state.
Reported: ms per MPC step, kernel launches per step (to_launch_count of every handle the loop uses), whether the two histories agree bit for
bit (NaN where both are), how many instances stayed finite, and the card's name and power limit, read in the same run.
    python profiles/mpc_bench.py [--T 50] [--runs 2] [--B 4096] [--out FILE]"""
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

WARM = 2     # untimed MPC steps before the timed ones (module loading, first allocations)


def zigzag_reference(p, nref, seed=7):
    """Xref[B, nref, n], Uref[B, nref, m]: hover at identity attitude along the zig-zag (0,-10,1) -> (10,0,1) -> (-10,0,1) -> (0,10,1), scaled
    to a tenth and travelled once over the reference, shifted per instance to start at its own initial position"""
    wp = 0.1 * np.array([[0, -10, 1.0], [10, 0, 1.0], [-10, 0, 1.0], [0, 10, 1.0]])
    s = np.linspace(0, len(wp) - 1, nref)
    i = np.minimum(s.astype(int), len(wp) - 2)
    path = wp[i] + (s - i)[:, None] * (wp[i + 1] - wp[i])
    Xref = np.zeros((p.B, nref, p.n))
    Xref[:, :, :3] = path[None] - path[0] + p.x0[:, None, :3]
    Xref[:, :, 3] = 1.0
    Xref[:, 1:, 7:10] = np.diff(Xref[:, :, :3], axis=1) / float(p.spec.dt[0])
    Uref = np.broadcast_to(TO.Quadrotor().hover_control(), (p.B, nref, p.m)).copy()
    return Xref, Uref


def launches(*ps):
    return sum(int(p._lib.to_launch_count(p._h)) for p in ps)


def device_arm(B, T, iters, Xref, Uref):
    p = problems.quadrotor(B=B, error_state=True)
    TO.mpc_setup(p, WARM + T, Xref=Xref, Uref=Uref)
    TO.mpc_run(p, WARM, iters)
    TO.mpc_history(p)
    l0 = launches(p)
    t0 = time.perf_counter()
    TO.mpc_run(p, T, iters)
    X, U, J = TO.mpc_history(p)                 # synchronises
    ms = (time.perf_counter() - t0) * 1e3 / T
    out = (ms, (launches(p) - l0) / T, (X, U, J))
    p.close()
    return out


def scripted_arm(B, T, iters, Xref, Uref):
    p = problems.quadrotor(B=B, error_state=True)
    obj = TO.LQRObjective(np.ones(p.n), np.ones(p.m), np.ones(p.n), np.zeros(p.n), 2)
    plant = TO.Problem(p.model, obj, p.x0, float(p.spec.dt[0]), error_state=True)
    X, U, J = [p.x0.copy()], [], []

    def step(j):
        TO.update_trajectory(p, Xref, Uref, 1 + j)
        TO.rollout(p)
        TO.ilqr_step(p, iters)
        u = TO.controls(p)[:, 0].copy()
        J.append(TO.merit(p).copy())
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
    out = (ms, (launches(p, plant) - l0) / T, (np.stack(X, 1), np.stack(U, 1), np.stack(J, 1)))
    p.close(); plant.close()
    return out


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
    for iters in (1, 3):
        for r in range(a.runs):
            d = device_arm(B, T, iters, Xref, Uref)
            s = scripted_arm(B, T, iters, Xref, Uref)
            same = all(np.array_equal(x, y, equal_nan=True) for x, y in zip(d[2], s[2]))   # an instance that diverged is NaN in both
            for name, arm in (("device", d), ("scripted", s)):
                entry = {"ms_per_step": round(arm[0], 3), "launches_per_step": arm[1]}
                res["runs"].setdefault(f"{name}_it{iters}", []).append(entry)
                print(f"{name} iterations={iters} run={r}", entry, flush=True)
            res["runs"].setdefault(f"bit_identical_it{iters}", []).append(bool(same))
            res["runs"].setdefault(f"finite_instances_it{iters}", []).append(int(np.all(np.isfinite(d[2][0]), axis=(1, 2)).sum()))
            print(f"iterations={iters} run={r} histories bit-identical: {same}", flush=True)
            if not same:   # where the two loops part: the first step of each history that differs, and in how many instances
                for name, x, y in zip("XUJ", d[2], s[2]):
                    bad = ~((x == y) | (np.isnan(x) & np.isnan(y)))
                    if bad.any():
                        at = np.argwhere(bad)
                        print(f"  {name}: first step {at[:, 1].min()}, {len(np.unique(at[:, 0]))} instances", flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
