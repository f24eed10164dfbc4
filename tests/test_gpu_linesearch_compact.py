"""The line search's knot loop for the compact problem class (forward.cu rollout_compact) against the loop every other fast-path problem
takes (rollout_fast), bit for bit.

The library built with -DTO_FWD_COMPACT=0 sends the compact class back to rollout_fast.  Each case runs once in a subprocess on each
library and the results must be identical: states, controls, merit J, max violation, alpha, line-search iterations and rho after a
rollout and several iterations (the late list is the set of instances whose ls_iters is above 4; it follows from ls_iters).  Bit-identity,
not a tolerance: the Quadrotor amplifies a last-bit difference to O(0.1) within six iterations (DESIGN.md 4a)."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANT = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "variants", "lib_fwd_loop.so")
DEFAULT = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "libtrajopt_b200.so")


def _quad(**kw):
    from trajopt_b200 import problems
    return problems.quadrotor(**kw)


def _per_instance_goals(p):
    import trajopt_b200 as TO
    rng = np.random.default_rng(3)
    xf = np.broadcast_to(np.asarray(p.xf, dtype=float), (p.B, p.n)).copy()
    xf[:, :3] += rng.uniform(-0.5, 0.5, (p.B, 3))
    TO.set_goal_state(p, xf)


def _tracking(p):
    import trajopt_b200 as TO
    X = np.asarray(TO.states(p)).copy()
    U = np.asarray(TO.controls(p))
    U = np.concatenate([U, U[:, -1:]], axis=1)      # [B, N, m]: the reference has as many control rows as state rows
    X[:, :, :3] += 0.1
    TO.update_trajectory(p, X, U)


def _state_bound(B, N):
    """a Bound on the state as well as the controls: the fast path, not the compact class"""
    import trajopt_b200 as TO
    n, m = 13, 4
    xf = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
    obj = TO.LQRObjective(np.full(n, 0.1), np.full(m, 0.01), np.full(n, 100.0), xf, N)
    cons = TO.ConstraintList(n, m, N)
    x_max = np.full(n, np.inf); x_max[2] = 2.5
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_max=x_max, u_min=np.zeros(m), u_max=np.full(m, 10.0)), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    rng = np.random.default_rng(1)
    x0 = np.broadcast_to(np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]), (B, n)).copy()
    x0[:, :3] += rng.uniform(-1, 1, (B, 3))
    p = TO.Problem(TO.Quadrotor(), obj, x0, 5.0, xf=xf, constraints=cons, error_state=True)
    TO.initial_controls(p, TO.Quadrotor().hover_control()[None, None, :] + 0.05 * rng.standard_normal((B, N - 1, m)))
    return p


def _per_knot_cost(B, N):
    """a different stage cost on every knot (a tracking objective built as one): not the compact class"""
    import trajopt_b200 as TO
    n, m = 13, 4
    xf = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
    Xr = np.linspace(np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]), xf, N)
    Ur = np.tile(TO.Quadrotor().hover_control(), (N - 1, 1))
    obj = TO.TrackingObjective(np.full(n, 0.1), np.full(m, 0.01), Xr, Ur, Qf=np.full(n, 100.0))
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=np.zeros(m), u_max=np.full(m, 10.0)), (1, N - 1))
    rng = np.random.default_rng(2)
    x0 = np.broadcast_to(Xr[0], (B, n)).copy()
    x0[:, :3] += rng.uniform(-1, 1, (B, 3))
    p = TO.Problem(TO.Quadrotor(), obj, x0, 5.0, xf=xf, constraints=cons, error_state=True)
    TO.initial_controls(p, Ur[None] + 0.05 * rng.standard_normal((B, N - 1, m)))
    return p


# name -> (factory, options, iterations, prepare, solve)
CASES = {
    "baseline_4096x101": (lambda: _quad(B=4096, N=101, error_state=True), {}, 4, None, False),
    "calm": (lambda: _quad(B=1024, N=101, error_state=True, u_noise=0.002), {}, 4, None, False),
    "fullstate": (lambda: _quad(B=512, N=101), {}, 4, None, False),
    "instance_goals": (lambda: _quad(B=512, N=101, error_state=True), {}, 4, _per_instance_goals, False),
    "tracking_reference": (lambda: _quad(B=512, N=101, error_state=True), {}, 4, _tracking, False),
    "ls_iters2": (lambda: _quad(B=512, N=101, error_state=True), dict(iterations_linesearch=2), 4, None, False),
    "ls_iters4": (lambda: _quad(B=512, N=101, error_state=True), dict(iterations_linesearch=4), 4, None, False),
    "ls_iters12": (lambda: _quad(B=512, N=101, error_state=True), dict(iterations_linesearch=12), 4, None, False),
    "N2": (lambda: _quad(B=256, N=2, error_state=True), {}, 3, None, False),
    "N3": (lambda: _quad(B=256, N=3, error_state=True), {}, 3, None, False),
    "N401": (lambda: _quad(B=256, N=401, error_state=True), {}, 3, None, False),
    "B1001": (lambda: _quad(B=1001, N=51, error_state=True), {}, 4, None, False),
    "solve": (lambda: _quad(B=256, N=51, error_state=True), {}, 0, None, True),
    # not the compact class: these take rollout_fast in both libraries
    "not_compact_state_bound": (lambda: _state_bound(256, 51), {}, 4, None, False),
    "not_compact_per_knot_cost": (lambda: _per_knot_cost(256, 51), {}, 4, None, False),
}


def run_case(name, out):
    """the worker: one case on the library LIBTRAJOPT_B200 names, results to the .npz `out`"""
    import trajopt_b200 as TO
    factory, opts, iters, prepare, solve = CASES[name]
    p = factory()
    if opts:
        TO.set_options(p, **opts)
    if prepare:
        prepare(p)
    res = {}
    TO.rollout(p)
    res["J0"] = TO.merit(p)
    if solve:
        st = TO.solve(p, iterations=60)
        for f in st.FIELDS:
            res["solve_" + f] = np.asarray(getattr(st, f))
    for i in range(iters):
        TO.ilqr_step(p, 1)
        s = TO.solver_state(p)
        for k in ("alpha", "ls_iters", "rho"):
            res[f"{k}{i}"] = s[k]
        res[f"J{i}"] = TO.merit(p)
        res[f"viol{i}"] = TO.max_violation(p)
    res["states"] = TO.states(p)
    res["controls"] = TO.controls(p)
    res["J"] = TO.merit(p)
    res["viol"] = TO.max_violation(p)
    np.savez(out, **res)
    p.close()


@pytest.fixture(scope="module")
def variant_lib(tmp_path_factory):
    if os.path.exists(VARIANT):
        return VARIANT
    d = str(tmp_path_factory.mktemp("variant"))
    subprocess.run(["bash", os.path.join(ROOT, "profiles", "scripts", "build_variant.sh"), "fwd_loop", "forward.cu", "-DTO_FWD_COMPACT=0"],
                   check=True, env=dict(os.environ, VARIANT_DIR=d), stdout=subprocess.DEVNULL)
    return os.path.join(d, "lib_fwd_loop.so")


def _run(lib, name, out):
    env = dict(os.environ, LIBTRAJOPT_B200=lib, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, "-s", os.path.abspath(__file__), name, out], check=True, env=env, cwd=ROOT)
    return dict(np.load(out))


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_compact_loop_is_bit_identical(case, variant_lib, tmp_path):
    new = _run(DEFAULT, case, str(tmp_path / "default.npz"))
    old = _run(variant_lib, case, str(tmp_path / "variant.npz"))
    assert sorted(new) == sorted(old)
    for k in old:
        assert new[k].dtype == old[k].dtype and new[k].shape == old[k].shape, k
        assert np.array_equal(new[k].view(np.uint8), old[k].view(np.uint8)), f"{case}: {k} differs between the two knot loops"
    if "ls_iters0" in new and case == "baseline_4096x101":
        assert np.any(new["ls_iters0"] > 4), "no instance reached the late passes"


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    run_case(sys.argv[1], sys.argv[2])
