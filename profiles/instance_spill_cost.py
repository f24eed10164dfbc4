"""Time of the per-instance (INST = true) kernel variants whose spills grew with the per-instance cost weights, on the paths they serve.

Every arm sets per-instance goals equal to the shared goal, so the INST = true kernels run on the shared numbers and the same work is timed
whichever build runs the script (run it from the parent's tree and from this one, alternated):
  quadrotor_nonfastal  full-state Quadrotor 4096 x 101 with a second control bound, so that a control entry has 4 AL rows and k_riccati<13, 4,
                       MMA> runs without the lane-resident AL terms: the backward phase;
  acrobot_fast         Acrobot with a DiagonalCost, 8192 x 201: the fast line search, the forward phase;
Reports ms per iLQR iteration with the per-phase CUDA-event timers, then, in a separate pass under torch.profiler, the mean device time of
each k_riccati, k_linesearch and k_cost kernel over 5 iterations and 10 rollout + to_merit calls (to_merit launches k_cost<merit, INST>).
    python profiles/instance_spill_cost.py [--steps 20] [--warmup 3]"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import trajopt_b200 as TO  # noqa: E402
from trajopt_b200 import _capi as K  # noqa: E402
from trajopt_b200 import problems  # noqa: E402
from instance_goals_bench import time_steps  # noqa: E402


def quadrotor_nonfastal():
    p = problems.quadrotor(B=4096, N=101, dt=0.05)
    TO.add_constraint(p.constraints, TO.BoundConstraint(13, 4, u_min=-50.0, u_max=50.0), (1, 100))
    TO.set_goal_state(p, np.tile(p.xf, (p.B, 1)))
    return p


def acrobot_fast():
    p = problems.acrobot(B=8192, N=201, dense_cost=False)
    TO.set_goal_state(p, np.tile(p.xf, (p.B, 1)))
    return p


def kernel_times(p):
    """mean device time (us) and launches of the backward, line-search and merit kernels, from a torch.profiler trace of their own pass"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        TO.ilqr_step(p, 5)
        for _ in range(10):
            TO.rollout(p)
            TO.merit(p)
        K.check(p._lib, p._h, p._lib.to_synchronize(p._h))
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if any(k in e.key for k in ("k_riccati", "k_linesearch", "k_cost")):
            total = getattr(e, "device_time_total", None) or e.cuda_time_total
            out[e.key[:120]] = [round(total / e.count, 2), e.count]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20); ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    res = {}
    for name, mk in (("quadrotor_nonfastal", quadrotor_nonfastal), ("acrobot_fast", acrobot_fast)):
        p = mk()
        ch = TO.kernel_choice(p)
        ms, ph = time_steps(p, a.steps, a.warmup)
        res[name] = {"backward": ch["backward"], "fastal": ch["fastal"], "linesearch": ch["linesearch"], "inst": ch["inst_backward"],
                     "ms_per_step": round(ms, 4), "phase_ms": ph}
        res[name]["kernel_us"] = kernel_times(p)
        p.close()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
