"""GPU parity under NON-DEFAULT solver options (`-m gpu`): the option values decide which code paths of the solver kernels run, and several
of those paths are unreachable with the defaults --

  A. the regularisation ladder of every backward kernel: restarts from rho = 0 and from bp_reg_initial > 0, a bp_reg_min large enough that
     the decrease zeroes rho, slow increase factors, failures at bp_reg_max.  For the register-resident kernel (riccati_frag.cu) that is
     every speculative round, the pool-slot and the recomputed winner, and the sequential tail past 15 restarts;
  B. the shapes of the parallel line search (forward.cu): pass 1 alone (iterations_linesearch < 4), one ladder pass (4..11), two (12..15);
     fast and generic rollouts, full state (no late list) and error state (late list), single stream and overlapped side stream;
  C. rejected trials (max_control_value / max_state_value), the failure commit, a non-default acceptance window, and failed backward
     passes going through the forward pass;
  D. the AL update with an active dual_max clamp, a non-default penalty_scaling and a reached penalty_max, and the reset of the
     regularisation that comes with every AL update, constrained or not.

Every group asserts, from the oracle's own results, the coverage it exists for, so that a change of inputs cannot quietly empty it."""
import numpy as np
import pytest

import trajopt_b200 as TO
from oracle_binding import OracleProblem, match_algebra
from parity_util import GAIN_TOL, check, decisions_agree, inst_err, triple_with_options

pytestmark = pytest.mark.gpu
P = TO.problems


# ---- the regularisation ladder, restated (Altro.jl regularization_update!; oracle.hpp reg_increase / reg_decrease) ---------------------
def reg_increase(o, rho, drho):
    drho = max(drho * o.bp_reg_increase_factor, o.bp_reg_increase_factor)
    return max(rho * drho, o.bp_reg_min), drho


def reg_decrease(o, rho, drho):
    drho = min(drho / o.bp_reg_increase_factor, 1.0 / o.bp_reg_increase_factor)
    return (rho * drho if rho * drho > o.bp_reg_min else 0.0), drho


def after_backward(o, rho, drho, status):
    """(rho, drho) after a backward pass that reported `status` restarts (-1: gave up at the first rho beyond bp_reg_max)"""
    if status >= 0:
        for _ in range(status):
            rho, drho = reg_increase(o, rho, drho)
        return reg_decrease(o, rho, drho)
    while True:
        rho, drho = reg_increase(o, rho, drho)
        if rho > o.bp_reg_max:
            return rho, drho


def failed_at(o, rho, drho):
    """the increase at which a failing backward pass starting from (rho, drho) gives up"""
    j = 0
    while True:
        j += 1
        rho, drho = reg_increase(o, rho, drho)
        if rho > o.bp_reg_max:
            return j


def between(f, j, lo=1e-8):
    """a bp_reg_max strictly between the j-th and (j+1)-th rho of the ladder from rho = 0, rho_j = lo f^(j(j+1)/2 - 1)"""
    return lo * f ** (j * (j + 1) / 2 - 1 + (j + 1) / 2)


def rel(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return float(np.max(np.abs(a - b) / np.maximum(1e-300, np.abs(b)), initial=0.0)) if np.all(np.isfinite(a)) else np.inf


def options(p):
    return p._options       # the complete option struct of the last set_options


# ---- A: backward-pass restarts and failures --------------------------------------------------------------------------------------------
def restart_problem(kind, B=64, N=21, seed=4):
    """a negative-definite control cost (R < 0): Quu + rho I is indefinite until rho has grown, so the ladder length follows from the
    options alone.  kind: compact error state (Goal/Bound, the record path), QuatVecEq error state (lie.cu), full state, small model"""
    def build(cls):
        r = np.random.default_rng(seed)
        if kind == "small":
            n, m = 4, 1
            stage = TO.DiagonalCost(np.ones(n), -0.5 * np.ones(m))
            term = TO.DiagonalCost(np.ones(n), -0.5 * np.ones(m), terminal=True)
            x0 = np.zeros((B, n)); x0[:, 1:3] = r.uniform(-0.5, 0.5, (B, 2))
            return cls(TO.Cartpole(), TO.Objective(stage, term, 11), x0, 0.5)
        n, m = 13, 4
        xf = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
        hover = TO.Quadrotor().hover_control()
        stage = TO.LQRCost(np.full(n, 0.1), np.full(m, -0.05), xf, hover)
        term = TO.LQRCost(np.full(n, 10.0), np.full(m, -0.05), xf, hover, terminal=True)
        cons = TO.ConstraintList(n, m, N)
        TO.add_constraint(cons, TO.BoundConstraint(n, m, u_min=np.zeros(4), u_max=np.full(4, 10.0)), (1, N - 1))
        if kind == "quatveceq":
            TO.add_constraint(cons, TO.QuatVecEq(n, m, xf[3:7]), N)
        x0 = np.tile(np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]), (B, 1))
        x0[:, :3] += r.uniform(-1, 1, (B, 3)); x0[:, 7:10] += r.uniform(-1, 1, (B, 3))
        p = cls(TO.Quadrotor(), TO.Objective(stage, term, N), x0, 1.0, xf=xf, constraints=cons, error_state=(kind != "full"))
        TO.initial_controls(p, hover + 0.05 * r.standard_normal((B, N - 1, m)))
        return p
    return build


RESTART_OPTIONS = [      # restarts of the compact error-state Quadrotor / of the Cartpole (the oracle's bp_status)
    dict(bp_reg_increase_factor=1.6),                                   # 9 / 9: the second speculative round of the fragment kernel
    dict(bp_reg_increase_factor=1.25),                                  # 12 / 13
    dict(bp_reg_increase_factor=1.1),                                   # 19 / 19: the sequential tail of the fragment kernel
    dict(bp_reg_initial=0.05),                                          # 2 / 3 from rho = 0.05: a first-round winner above the lowest candidate
    dict(bp_reg_initial=1e-3),                                          # 5 / 5
    dict(bp_reg_min=0.2),                                               # 1 / 3, and the decrease after the pass zeroes rho (rho f^-1 < bp_reg_min)
    dict(bp_reg_min=1.0),                                               # 1 / 1
    dict(bp_reg_initial=1.0),                                           # 0 / 0
    dict(bp_reg_max=between(1.6, 0)),                                   # bp_reg_max < bp_reg_min: gives up at the first increase
    dict(bp_reg_max=between(1.6, 2)),                                   # gives up at the 3rd increase (first round of the fragment kernel)
    dict(bp_reg_max=between(1.6, 6)),                                   # ... at the 7th (second round)
    dict(bp_reg_increase_factor=1.1, bp_reg_max=between(1.1, 17)),      # ... at the 18th (sequential tail)
]

RESTART_KERNELS = {                # name: (problem kind, backward_kernel, to_backward_algebra)
    "frag": ("compact", None, 1),
    "compact_kernel5": ("compact", 5, 0),
    "compact_kernel3": ("compact", 3, 0),
    "quatveceq_lie": ("quatveceq", None, 0),
    "fullstate": ("full", None, 0),
    "small_kernel1": ("small", 1, 0),
    "small_kernel2": ("small", 2, 0),
}


def backward_pair(g, o, frag):
    sg, so = TO.backward(g), TO.backward(o)
    if frag:
        g._call("to_synchronize")       # a queue overflow / spin-limit error of the fragment kernel is reported here
    return sg, so


def run_restarts(build, opts, kernel, algebra, frag):
    """one backward pass (and a second one from the regularisation state the first left) against the oracle and the closed form"""
    g, o = build(TO.Problem), build(OracleProblem)
    TO.set_options(g, **opts, **({} if kernel is None else {"backward_kernel": kernel}))
    TO.set_options(o, **opts)
    match_algebra(g, o)
    assert TO.backward_algebra(g) == algebra
    oo = options(o)
    for p in (g, o):
        TO.rollout(p); TO.expand(p)
    rho0 = TO.solver_state(o)["rho"]
    assert np.all(rho0 == oo.bp_reg_initial)
    sg, so = backward_pair(g, o, frag)
    assert np.array_equal(sg, so), f"restarts {opts}: cuda {np.unique(sg)} oracle {np.unique(so)}"
    stg, sto = TO.solver_state(g), TO.solver_state(o)
    closed = [after_backward(oo, rho0[b], 0.0, so[b]) for b in range(g.B)]
    assert rel(sto["rho"], [c[0] for c in closed]) <= 1e-12, "oracle rho vs the closed form of the ladder"
    assert rel(stg["rho"], sto["rho"]) <= 1e-12, f"rho after the pass {opts}"
    assert rel(stg["rho"], [c[0] for c in closed]) <= 1e-12, f"rho vs the closed form {opts}"
    ok = so >= 0
    errs = [0.0]
    if ok.any():
        (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
        for what, a, b in (("K", Kg, Ko), ("d", dg, do), ("dV", stg["dV"], sto["dV"])):
            e = inst_err(a[ok], b[ok])
            assert e.max() <= GAIN_TOL, f"{what} after restarts {opts}: {e.max():.3e}"
            errs.append(float(e.max()))
    sg2, so2 = backward_pair(g, o, frag)        # from the rho / drho the first pass left: checks drho, which is not exported
    assert np.array_equal(sg2, so2), f"restarts of the second pass {opts}"
    closed2 = [after_backward(oo, c[0], c[1], s) for c, s in zip(closed, so2)]
    assert rel(TO.solver_state(g)["rho"], TO.solver_state(o)["rho"]) <= 1e-12, f"rho after the second pass {opts}"
    assert rel(TO.solver_state(g)["rho"], [c[0] for c in closed2]) <= 1e-12, f"rho after the second pass vs the closed form {opts}"
    fails = [failed_at(oo, rho0[b], 0.0) for b in range(g.B) if so[b] < 0]
    g.close(); o.close()
    return so, fails, max(errs)


def test_ladder_closed_form():
    """the restated ladder from rho = 0 is rho_j = bp_reg_min f^(j(j+1)/2 - 1) (needs no oracle), and `between` separates two steps of it"""
    class O:
        bp_reg_min, bp_reg_max = 1e-8, 1e8
    for f in (1.6, 1.25, 1.1):
        O.bp_reg_increase_factor = f
        rho, drho = 0.0, 0.0
        for j in range(1, 25):
            rho, drho = reg_increase(O, rho, drho)
            assert abs(rho - 1e-8 * f ** (j * (j + 1) / 2 - 1)) <= 1e-12 * rho
            assert 1e-8 * f ** (j * (j + 1) / 2 - 1) < between(f, j) < 1e-8 * f ** ((j + 1) * (j + 2) / 2 - 1)


@pytest.mark.parametrize("name", sorted(RESTART_KERNELS))
def test_backward_restarts_and_failures_match_oracle(name):
    kind, kernel, algebra = RESTART_KERNELS[name]
    frag = name == "frag"
    statuses, fails, worst = [], [], 0.0
    for opts in RESTART_OPTIONS:
        so, fl, e = run_restarts(restart_problem(kind), opts, kernel, algebra, frag)
        statuses.append(so); fails += fl; worst = max(worst, e)
    s = np.concatenate(statuses)
    bands = {"0": s == 0, "1": s == 1, "2-3": (s >= 2) & (s <= 3), "4-7": (s >= 4) & (s <= 7), "8-15": (s >= 8) & (s <= 15), ">=16": s >= 16,
             "failed": s < 0}
    assert all(v.any() for v in bands.values()), {k: int(v.sum()) for k, v in bands.items()}
    fails = np.array(fails)
    # failures inside every speculative round of the fragment kernel ({1..3}, {4..15}) and inside its sequential tail
    assert np.any(fails == 1) and np.any((fails >= 2) & (fails <= 3)) and np.any((fails >= 4) & (fails <= 15)) and np.any(fails >= 16), np.unique(fails)
    print(f"{name}: worst gain / dV error {worst:.2e}")


@pytest.mark.parametrize("opts,N", [(dict(bp_reg_increase_factor=1.6), 16), (dict(bp_reg_initial=0.05), 21)], ids=["round2_winner", "round1_winner"])
def test_fragment_kernel_restarts_beyond_the_pool(opts, N):
    """more instances than pool slots (4096), each restarting at least twice: winners above the lowest candidate of their round come from a
    pool slot or, without one, from one more sweep -- both happen in one launch.  (The horizons keep every winning rho clear of the
    threshold of its instance: where Quu + rho I is only just definite the gains are ill-conditioned, and even the oracle's two arithmetic
    forms of the backward pass differ by 1e-7 -- at N = 21, f = 1.6 on these inputs.)"""
    build = restart_problem("compact", B=4200, N=N)
    so, fails, e = run_restarts(build, opts, None, 1, True)
    assert np.all(so >= 2) and not fails and len(np.unique(so)) == 1
    if "bp_reg_initial" not in opts:
        assert np.all(so >= 8)
    print(f"B = 4200, {so[0]} restarts: worst gain error {e:.2e}")


# ---- B: the shapes of the parallel line search ---------------------------------------------------------------------------------------
LS_PROBLEMS = {     # fast path: diagonal cost + Goal/Bound; generic path: dense cost.  Error state + fast path = the record path (late list).
    "fast_full": lambda cls: P.quadrotor(B=48, N=21, dt=0.05, cls=cls),
    "fast_errstate": lambda cls: P.quadrotor(B=48, N=21, dt=0.05, error_state=True, cls=cls),
    "generic_full": lambda cls: P.quadrotor(B=48, N=21, dt=0.05, dense_cost=True, cls=cls),
    "generic_errstate": lambda cls: P.quadrotor(B=48, N=21, dt=0.05, dense_cost=True, error_state=True, cls=cls),
}


def iterate(trio, driver, iters=1):
    for _ in range(iters):
        for p in trio:
            if driver == "ilqr_step":
                TO.ilqr_step(p, 1)          # the later passes on the overlapped side stream (full state, record path)
            else:
                TO.expand(p); TO.backward(p); TO.forward(p)      # everything on one stream


def compare_iterates(trio, what, outliers=0.0):
    g, o, t = trio
    sg, so, st = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    dec = (so["alpha"] == st["alpha"]) & (so["ls_iters"] == st["ls_iters"]) & (so["bp_status"] == st["bp_status"])
    for k in ("bp_status", "alpha", "ls_iters"):
        decisions_agree(f"{what}: {k}", sg[k], so[k], st[k], allow=0.05)
    same = dec & (sg["alpha"] == so["alpha"]) & (sg["ls_iters"] == so["ls_iters"]) & (sg["bp_status"] == so["bp_status"])
    e = [check(f"{what}: rho", sg["rho"], so["rho"], st["rho"], 1e-12, same, outliers)[0],
         check(f"{what}: J", TO.merit(g), TO.merit(o), TO.merit(t), 1e-9, same, outliers)[0],
         check(f"{what}: X", TO.states(g), TO.states(o), TO.states(t), 1e-9, same, outliers)[0],
         check(f"{what}: U", TO.controls(g), TO.controls(o), TO.controls(t), 1e-9, same, outliers)[0]]
    return so, max(e)


@pytest.mark.parametrize("driver", ["forward", "ilqr_step"])
@pytest.mark.parametrize("path", sorted(LS_PROBLEMS))
@pytest.mark.parametrize("L", [0, 1, 3, 4, 5, 11, 12, 15])
def test_line_search_shapes_match_oracle(L, path, driver):
    """iterations_linesearch decides the passes: < 4 pass 1 commits failures, 4..11 one ladder pass, 12..15 two.  A control envelope
    (max_control_value just above hover) rejects the long steps of a poor first guess, so the accepted trial spreads over the whole ladder."""
    opts = dict(iterations_linesearch=L, max_control_value=1.5 if L >= 4 else 3.0)
    trio = triple_with_options(LS_PROBLEMS[path], opts)
    for p in trio:
        TO.rollout(p)
    iterate(trio, "ilqr_step", 2)
    iterate(trio, driver)
    so, e = compare_iterates(trio, f"L={L} {path} {driver}")
    ls, acc = so["ls_iters"], so["alpha"] > 0
    assert np.all((ls >= 1) & (ls <= L + 1))
    assert np.any(acc) and (np.any(~acc & (ls == L + 1)) or L == 15), np.bincount(ls)      # accepted steps, and failures
    if L >= 4:
        assert np.any(ls > 4), np.bincount(ls)
    if L >= 12:
        assert np.any(ls > 12), np.bincount(ls)
    for p in trio:
        p.close()
    print(f"L={L} {path} {driver}: ls_iters {np.bincount(ls, minlength=L + 2)}, worst error {e:.2e}")


# ---- C: rejected trials, the failure commit, the acceptance window, failed backward passes ---------------------------------------------
@pytest.mark.parametrize("driver", ["forward", "ilqr_step"])
@pytest.mark.parametrize("path", ["fast_full", "fast_errstate", "generic_full"])
@pytest.mark.parametrize("L", [3, 10, 12])
def test_forced_line_search_failure(L, path, driver):
    """max_control_value below the hover thrust rejects every trial: alpha = 0, ls_iters = L + 1, rho = reg_increase(rho) + bp_reg_fp, and the
    trajectory stays bit for bit"""
    g, o, t = triple_with_options(LS_PROBLEMS[path], dict(iterations_linesearch=L, max_control_value=0.5))
    for p in (g, o):
        TO.rollout(p)
    X0, U0 = TO.states(g), TO.controls(g)
    Xo, Uo = TO.states(o), TO.controls(o)
    iterate((g, o), driver)
    opt = options(o)
    for p, X, U in ((g, X0, U0), (o, Xo, Uo)):
        s = TO.solver_state(p)
        assert np.all(s["alpha"] == 0) and np.all(s["ls_iters"] == L + 1) and np.all(s["bp_status"] >= 0)
        assert np.array_equal(TO.states(p), X) and np.array_equal(TO.controls(p), U)
    so = TO.solver_state(o)["bp_status"]
    assert np.array_equal(TO.solver_state(g)["bp_status"], so)
    expect = []
    for b in range(g.B):
        rho, drho = after_backward(opt, opt.bp_reg_initial, 0.0, so[b])
        rho, drho = reg_increase(opt, rho, drho)
        expect.append(rho + opt.bp_reg_fp)
    assert rel(TO.solver_state(o)["rho"], expect) <= 1e-15
    assert rel(TO.solver_state(g)["rho"], expect) <= 1e-12
    for p in (g, o, t):
        p.close()


def probe_accepted(build):
    """the oracle's accepted first step with default options: per-instance max |u| and max |x_{k >= 2}| of its trajectory, and ls_iters"""
    p = build(OracleProblem)
    TO.rollout(p); TO.expand(p); TO.backward(p); TO.forward(p)
    s = TO.solver_state(p)
    U, X = TO.controls(p), TO.states(p)
    out = np.abs(U).max(axis=(1, 2)), np.abs(X[:, 1:]).max(axis=(1, 2)), s["ls_iters"].copy()
    p.close()
    return out


@pytest.mark.parametrize("which", ["max_control_value", "max_state_value"])
@pytest.mark.parametrize("path", ["fast_full", "fast_errstate", "generic_full"])
def test_partial_rejection_matches_oracle(path, which):
    """an envelope set from the oracle's own accepted steps: the instances whose step leaves it backtrack further (or fail), the others keep
    their step"""
    build = LS_PROBLEMS[path]
    umax, xmax, ls0 = probe_accepted(build)
    bound = float(np.median(umax if which == "max_control_value" else xmax))
    trio = triple_with_options(build, {which: bound})
    for p in trio:
        TO.rollout(p)
    iterate(trio, "forward")
    so, e = compare_iterates(trio, f"{which} = {bound:.4g} {path}")
    ls = so["ls_iters"]
    assert np.any(ls > ls0) and np.any((so["alpha"] > 0) & (ls == ls0)) and np.any((so["alpha"] > 0) & (ls > ls0)), (ls0, ls)
    for p in trio:
        p.close()
    print(f"{which} {path}: worst error {e:.2e}")


@pytest.mark.parametrize("window", [(-1.0, 10.0), (-3.0, -0.2)], ids=["negative_lower", "negative_window"])
@pytest.mark.parametrize("path", ["fast_full", "fast_errstate", "generic_full"])
def test_acceptance_window_matches_oracle(path, window):
    """lower < z <= upper or J < J_prev: a negative lower bound accepts some increases of the cost; a negative upper bound
    also rejects the small increases"""
    lo, hi = window
    build = LS_PROBLEMS[path]
    trio = triple_with_options(lambda cls: _poor_guess(build, cls), dict(line_search_lower_bound=lo, line_search_upper_bound=hi))
    for p in trio:
        TO.rollout(p)
    J0 = TO.merit(trio[1])
    iterate(trio, "forward")
    so, e = compare_iterates(trio, f"window ({lo}, {hi}] {path}")
    J1 = TO.merit(trio[1])
    assert np.any((so["alpha"] > 0) & (J1 > J0)), "no accepted increase of the cost"
    # the same inputs with the default window take other decisions
    ref = _poor_guess(build, OracleProblem)
    TO.rollout(ref); TO.expand(ref); TO.backward(ref); TO.forward(ref)
    assert np.any(TO.solver_state(ref)["ls_iters"] != so["ls_iters"])
    ref.close()
    for p in trio:
        p.close()
    print(f"window ({lo}, {hi}] {path}: worst error {e:.2e}")


def _poor_guess(build, cls):
    p = build(cls)
    r = np.random.default_rng(7)
    TO.initial_controls(p, TO.controls(p) + 1.5 * r.standard_normal((p.B, p.N - 1, p.m)))
    return p


@pytest.mark.parametrize("driver", ["forward", "ilqr_step"])
@pytest.mark.parametrize("path", ["fast_full", "fast_errstate"])
def test_failed_backward_pass_keeps_trajectory(path, driver):
    """a backward pass that gives up (status -1) leaves its instance to the forward pass with alpha = 0, ls_iters = 0 and the trajectory
    unchanged -- on the overlapped path too, where that instance is not accepted by pass 1 and goes through the late list"""
    build = restart_problem("compact" if path == "fast_errstate" else "full")
    g, o, t = triple_with_options(build, dict(bp_reg_max=between(1.6, 7)))      # every instance needs 10 restarts: all give up at 8
    for p in (g, o, t):
        TO.rollout(p)
    X0, U0 = TO.states(g), TO.controls(g)
    iterate((g, o, t), driver)
    sg, so = TO.solver_state(g), TO.solver_state(o)
    assert np.all(so["bp_status"] == -1)
    assert np.array_equal(sg["bp_status"], so["bp_status"])
    for s in (sg, so):
        assert np.all(s["alpha"] == 0) and np.all(s["ls_iters"] == 0)
    assert np.array_equal(TO.states(g), X0) and np.array_equal(TO.controls(g), U0)
    assert rel(sg["rho"], so["rho"]) <= 1e-12
    for p in (g, o, t):
        p.close()


@pytest.mark.parametrize("driver", ["forward", "ilqr_step"])
def test_failed_backward_pass_among_accepted_instances(driver):
    """the record path with a bp_reg_max that some instances of a poor first guess exceed and others do not"""
    build = lambda cls: P.quadrotor(B=64, N=21, dt=0.05, error_state=True, u_noise=2.0, cls=cls)
    g, o, t = triple_with_options(build, dict(bp_reg_max=between(1.6, 7)))
    for p in (g, o, t):
        TO.rollout(p)
    X0, U0 = TO.states(g), TO.controls(g)
    iterate((g, o, t), driver)
    sg, so = TO.solver_state(g), TO.solver_state(o)
    failed = so["bp_status"] < 0
    assert failed.any() and (~failed).any() and np.any(so["alpha"][~failed] > 0)
    decisions_agree("bp_status", sg["bp_status"], so["bp_status"], TO.solver_state(t)["bp_status"])
    f = failed & (sg["bp_status"] < 0)
    assert f.sum() >= 0.9 * failed.sum()
    assert np.all(sg["alpha"][f] == 0) and np.all(sg["ls_iters"][f] == 0)
    assert np.array_equal(TO.states(g)[f], X0[f]) and np.array_equal(TO.controls(g)[f], U0[f])
    # (one accepted instance of this poor first guess sits outside the budget of the comparison of its step: allow one in twenty)
    compare_iterates((g, o, t), f"bp failures {driver}", outliers=0.05)
    for p in (g, o, t):
        p.close()


# ---- D: the AL update ------------------------------------------------------------------------------------------------------------------
def al_problem(cls):
    """Quadrotor with bounds, goal and a second-order-cone norm on the controls that the hover thrust violates"""
    base = P.quadrotor(B=16, N=21, dt=0.05, cls=cls)
    n, m, N = 13, 4, 21
    cons = base.constraints
    TO.add_constraint(cons, TO.NormConstraint(n, m, 2.0, TO.SecondOrderCone(), "control"), (1, N - 1))
    p = cls(base.model, base.obj, base.x0, 1.0, xf=base.xf, constraints=cons)
    TO.initial_controls(p, TO.controls(base)); base.close()
    return p


def test_al_update_clamp_and_penalty_cap_match_oracle():
    dual_max, rho_init = 0.5, 0.01
    trio = triple_with_options(al_problem, dict(dual_max=dual_max, penalty_scaling=3.0, penalty_max=7.0, bp_reg_initial=rho_init))
    g, o, t = trio
    for p in trio:
        TO.rollout(p); TO.ilqr_step(p, 2)
    clamped = np.zeros(3, dtype=bool)
    worst = 0.0
    for update, mu in ((1, 3.0), (2, 7.0)):
        for p in trio:
            TO.al_update(p)
        for p in (g, o):
            assert np.all(TO.solver_state(p)["rho"] == rho_init), "the AL update restarts the regularisation"
        sg, so, st = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
        for i in range(3):
            lo = TO.multipliers(o, i)
            assert np.all(np.abs(lo) <= dual_max)
            clamped[i] |= np.any(np.abs(lo) == dual_max)
            worst = max(worst, check(f"multipliers {i} after update {update}", TO.multipliers(g, i), lo, TO.multipliers(t, i), 1e-9)[0])
            assert TO.penalty(g, i) == TO.penalty(o, i) == mu       # 1 -> 3 -> min(9, penalty_max)
        worst = max(worst, check(f"merit after update {update}", TO.merit(g), TO.merit(o), TO.merit(t), 1e-9)[0])
        for p in trio:
            TO.ilqr_step(p, 2)
        _, e = compare_iterates(trio, f"2 iterations after update {update}")
        worst = max(worst, e)
    assert clamped.all(), f"dual_max clamp active on (bound, goal, SOC) = {clamped}"
    for p in trio:
        p.close()
    print(f"AL update: worst error {worst:.2e}")


@pytest.mark.parametrize("name", ["cartpole", "quadrotor_unconstrained", "quadrotor_errstate"])
def test_al_update_resets_regularisation(name):
    """Altro's inner solve starts every AL iteration from bp_reg_initial: to_al_update resets rho / drho on every instance, whether the
    problem has constraints or not (an unconstrained problem has no multipliers to update, but its regularisation restarts all the same)"""
    build = {"cartpole": lambda cls: P.cartpole(B=16, N=51, cls=cls),
             "quadrotor_unconstrained": lambda cls: P.quadrotor(B=16, N=21, dt=0.05, constrained=False, cls=cls),
             "quadrotor_errstate": lambda cls: P.quadrotor(B=16, N=21, dt=0.05, error_state=True, cls=cls)}[name]
    rho_init = 0.01
    trio = triple_with_options(build, dict(bp_reg_initial=rho_init))
    g, o, t = trio
    for p in trio:
        TO.rollout(p); TO.ilqr_step(p, 3)
    assert np.any(TO.solver_state(o)["rho"] != rho_init)       # the iterations moved rho off its initial value
    for p in trio:
        TO.al_update(p)
    for p in (g, o):
        assert np.all(TO.solver_state(p)["rho"] == rho_init)
    for p in trio:
        TO.ilqr_step(p, 2)       # from the reset drho: the ladder of these iterations restarts too
    compare_iterates(trio, f"{name}: 2 iterations after the AL update")
    for p in trio:
        p.close()
