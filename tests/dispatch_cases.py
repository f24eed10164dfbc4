"""Problems one step either side of every shape-driven kernel choice of the solver (the table of DESIGN.md 4a), and a plain-Python
restatement of the predicates that make those choices -- test infrastructure shared by tests/test_dispatch_cases.py (CPU: each pair
straddles its threshold, the oracle runs both sides) and tests/test_gpu_dispatch_boundaries.py (each side lands on the kernel it was
built for, and matches the oracle there).

Every builder takes the Problem class (CUDA or oracle) and returns the same problem for both.  The restatement mirrors, constant for
constant, the launch-time predicates of csrc/forward.cu (linesearch_path), riccati.cu (backward_plan: the backward kernel, FASTAL and
the records' term table), riccati_small.cu (riccati_small_supported), riccati_frag.cu and capi.cu (to_create's problem flags);
`to_kernel_choice` reports what the library itself decided.  A change to one of those constants has to move the matching case here."""
from dataclasses import dataclass, field

import numpy as np

import trajopt_b200 as TO

# the thresholds, as the library has them
FWD_MAX_N = 512          # forward.cu: FwdTab::dt / cost_index / lam_off / lam_cnt
FWD_MAX_COST = 4         # forward.cu: costs cached in shared memory
MAXT = 3                 # common.cuh TO_EXP_MAXT: lane-resident AL terms per z entry (FASTAL); the records' term table (rec_fused)
MAXP_KNOT_PACKED = 128   # riccati.cu backward_plan: rows per knot of the packed term fields (FASTAL, rec_fused)
SOLVER_MAXP = 16         # capi.cu solver_supported: rows per general constraint in the solver kernels
CREATE_MAXP = 32         # capi.cu build_con (TO_MAXP): rows per general constraint
SMALL_WAVE = 16          # riccati_small.cu: the thread kernel past 16 one-warp CTAs per SM
SMS_H100 = 132           # SM count the CPU suite assumes (the GPU tests read the device's)
RESIDENT_H100 = 2112     # k_riccati_frag warps resident at once on 132 SMs (4 CTAs of 4 warps per SM); the GPU tests read the library's

LINESEARCH = ("generic", "fast", "compact")
BACKWARD = ("thread", "warp_mma", "warp_dfma", "fragment", "dense_mma", "dense_dfma")

QXF = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
QX0 = np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
HOVER = TO.Quadrotor().hover_control()


# ---- the restatement ------------------------------------------------------------------------------------------------------------

def _diag_cost(c):
    return bool(getattr(c, "is_diag", False)) and not isinstance(c, (TO.DiagonalQuatCost, TO.AutodiffCost))


def features(prob):
    """the problem flags to_create derives (capi.cu), from the Python description alone"""
    n, m, N = prob.n, prob.m, prob.N
    uniq, index = prob.obj._tables()
    cons = list(zip(prob.constraints.inds, prob.constraints.constraints))
    diag = [isinstance(c, (TO.GoalConstraint, TO.BoundConstraint)) for _, c in cons]
    f = dict(n=n, m=m, N=N, B=prob.B, lie=bool(prob.error_state), ne=prob.ne, ncost=len(uniq),
             all_diag_cost=all(_diag_cost(c) for c in uniq), all_diag_con=all(diag),
             special_cost=any(isinstance(c, (TO.DiagonalQuatCost, TO.AutodiffCost)) for c in uniq))
    terms = np.zeros(n + m, dtype=int)
    for (_, c), d in zip(cons, diag):
        if isinstance(c, TO.GoalConstraint):
            terms[np.asarray(c.inds) - 1] += 1
        elif d:
            terms += np.isfinite(c.z_max).astype(int) + np.isfinite(c.z_min).astype(int)
    f["max_terms_per_z"] = int(terms.max())
    pk = [sum(c.p for (a, b), c in cons if a <= k <= b) for k in range(1, N + 1)]
    nk = [sum(1 for (a, b), c in cons if a <= k <= b) for k in range(1, N + 1)]
    f["max_p_knot"], f["max_cons_knot"] = max(pk), max(nk)
    f["max_general_p"] = max([c.p for (_, c), d in zip(cons, diag) if not d], default=0)
    cls = N >= 2 and f["all_diag_cost"] and f["all_diag_con"] and all(index[k] == index[0] for k in range(1, N - 1))
    nbox = ngoal = 0
    for (a, b), c in cons:
        if isinstance(c, TO.BoundConstraint):
            on_u = np.arange(n + m) >= n
            cls = cls and a == 1 and b == N - 1 and c.p == 2 * m and np.array_equal(np.isfinite(c.z_max), on_u) \
                and np.array_equal(np.isfinite(c.z_min), on_u)
            nbox += 1
        elif isinstance(c, TO.GoalConstraint):
            cls = cls and a == N and b == N
            ngoal += 1
        else:
            cls = False
    f["fwd_compact"] = bool(cls and nbox <= 1 and ngoal <= 1)
    f["dense_riccati"] = f["lie"] or f["special_cost"]
    f["compact"] = f["lie"] and all(_diag_cost(c) for c in uniq) and f["all_diag_con"] and f["ne"] == 12 and m == 4
    return f


def predicted(prob, backward_kernel=0, sms=SMS_H100):
    """the kernel choice the library should report for `prob` (to_kernel_choice, TO.kernel_choice), restated"""
    f = features(prob)
    n, m = f["n"], f["m"]
    fast = f["all_diag_cost"] and f["all_diag_con"] and f["N"] <= FWD_MAX_N and f["max_p_knot"] <= 2 * (n + m) and f["max_cons_knot"] <= 2
    compact = fast and f["fwd_compact"] and f["ncost"] <= FWD_MAX_COST
    ls = "compact" if compact else ("fast" if fast else "generic")
    record = f["compact"] and backward_kernel not in (3, 5)
    if record:
        bk = "fragment"
    elif f["dense_riccati"]:
        bk = "dense_mma" if (f["ne"] == 12 and m == 4 and backward_kernel != 3) else "dense_dfma"
    else:
        small = n <= 4 and m <= 2 and f["all_diag_con"]
        if small and (backward_kernel == 2 or (backward_kernel == 0 and f["B"] > SMALL_WAVE * sms)):
            bk = "thread"
        else:
            bk = "warp_mma" if (n >= 8 and m <= 4 and f["all_diag_cost"] and f["all_diag_con"]) else "warp_dfma"
    packed = f["max_terms_per_z"] <= MAXT and f["N"] < 4095 and f["max_p_knot"] < MAXP_KNOT_PACKED
    return dict(linesearch=ls, cost_cached=ls != "generic" and f["ncost"] <= FWD_MAX_COST, backward=bk,
                fastal=bk in ("warp_mma", "warp_dfma") and packed, rec_fused=record and packed, late_list=f["compact"])


def solver_accepts(prob):
    return features(prob)["max_general_p"] <= SOLVER_MAXP


def create_accepts(prob):
    return features(prob)["max_general_p"] <= CREATE_MAXP


# ---- builders -------------------------------------------------------------------------------------------------------------------

def _quad(cls, obj, cons, B, N, seed, error_state=False, dt=0.05):
    r = np.random.default_rng(seed)
    x0 = np.tile(QX0, (B, 1)); x0[:, :3] += r.uniform(-1, 1, (B, 3))
    p = cls(TO.Quadrotor(), obj, x0, dt * (N - 1), xf=QXF, constraints=cons, error_state=error_state)
    TO.initial_controls(p, HOVER + 0.05 * r.standard_normal((B, N - 1, 4)))
    return p


def _qcost(w=0.1, terminal=False):
    return TO.LQRCost(np.full(13, 100.0 if terminal else w), np.full(4, 0.01), QXF, HOVER, terminal=terminal)


def _box(cons, N, lo=0.0, hi=10.0, knots=None):
    TO.add_constraint(cons, TO.BoundConstraint(13, 4, u_min=np.full(4, lo), u_max=np.full(4, hi)), knots or (1, N - 1))


def _pos_bound(upper=(2.4, 2.6, 2.4), lower=None):
    x_max, x_min = np.full(13, np.inf), np.full(13, -np.inf)
    x_max[:3] = upper
    if lower is not None:
        x_min[:3] = lower
    return TO.BoundConstraint(13, 4, x_min=x_min, x_max=x_max)


def horizon(cls, N, error_state=False, B=4):
    """F1: a position bound on knots 2..N beside the control box and the goal (not the compact class, so the fast loop reads FwdTab)"""
    cons = TO.ConstraintList(13, 4, N)
    TO.add_constraint(cons, _pos_bound(), (2, N))
    _box(cons, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    return _quad(cls, TO.Objective(_qcost(), _qcost(terminal=True), N), cons, B, N, seed=21, error_state=error_state, dt=0.01)


def overlap(cls, third, B=8, N=41):
    """F2: constraints inserted Goal (N), position bound (20..N), control box (1..N-1): knots 20..N-1 stage the bound's multipliers before
    the box's, knot N the goal's before the bound's.  `third`: a goal on the attitude at knot 30, three constraints there"""
    cons = TO.ConstraintList(13, 4, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    TO.add_constraint(cons, _pos_bound(), (20, N))
    _box(cons, N)
    if third:
        TO.add_constraint(cons, TO.GoalConstraint(QXF, inds=[4, 5, 6]), 30)
    return _quad(cls, TO.Objective(_qcost(), _qcost(terminal=True), N), cons, B, N, seed=22)


def rows_per_knot(cls, extra, B=8, N=31):
    """F3: DoubleIntegrator 2-D (2(n+m) = 12) with every z entry bounded on both sides on knots 1..N-1 -- 12 rows, the stage's multiplier
    slots exactly full -- and the goal at N; `extra`: one more row (a goal on x1) at knot 10"""
    n, m = 4, 2
    xf = np.array([0, 2.0, 0, 0])
    obj = TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n) * (N - 1), xf, N)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.BoundConstraint(n, m, x_min=np.full(n, -5.0), x_max=np.full(n, 5.0), u_min=-4.0, u_max=4.0), (1, N - 1))
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    if extra:
        TO.add_constraint(cons, TO.GoalConstraint(xf, inds=[1]), 10)
    r = np.random.default_rng(23)
    p = cls(TO.DoubleIntegrator(2), obj, 0.3 * r.standard_normal((B, n)), 3.0, xf=xf, constraints=cons)
    TO.initial_controls(p, r.standard_normal((B, N - 1, m)))
    return p


def costs(cls, ncost, B=8, N=41):
    """F4: `ncost` distinct diagonal costs (ncost - 1 stage costs on consecutive knot blocks + the terminal cost), box + goal"""
    stage = [_qcost(0.1 + 0.05 * j) for j in range(ncost - 1)]
    per = [stage[min(k * (ncost - 1) // (N - 1), ncost - 2)] for k in range(N - 1)]
    cons = TO.ConstraintList(13, 4, N)
    _box(cons, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    return _quad(cls, TO.Objective(per, _qcost(terminal=True)), cons, B, N, seed=24)


COMPACT_FLIPS = ("member", "one_sided_box", "box_short", "goal_early", "second_box", "stage_cost")


def compact(cls, flip, B=8, N=31):
    """F5: the BASELINE problem (the compact class) and each of its membership conditions flipped alone"""
    stage, term = _qcost(), _qcost(terminal=True)
    per = [stage] * (N - 1)
    if flip == "stage_cost":
        per[4] = _qcost(0.2)
    cons = TO.ConstraintList(13, 4, N)
    if flip == "one_sided_box":
        TO.add_constraint(cons, TO.BoundConstraint(13, 4, u_min=np.zeros(4)), (1, N - 1))
    else:
        _box(cons, N, knots=(2, N - 1) if flip == "box_short" else None)
    if flip == "second_box":
        _box(cons, N, lo=0.5, hi=9.0)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N - 1 if flip == "goal_early" else N)
    return _quad(cls, TO.Objective(per, term), cons, B, N, seed=25)


SMALL_MODELS = ("cartpole", "acrobot", "double_integrator")


def small(cls, model, B, N=51, general=False):
    """R1 / R2: the small models with a control box and a goal; `general`: plus one LinearConstraint on the state (a general constraint)"""
    if model == "cartpole":
        p = TO.problems.cartpole(B=B, N=N, u_bound=3.0, goal=True, cls=cls)
    elif model == "acrobot":
        p = TO.problems.acrobot(B=B, N=N, cls=cls)
    else:
        p = TO.problems.double_integrator(B=B, N=N, dim=2, cls=cls)
    if general:
        A = np.zeros((1, p.n)); A[0, 0] = 1.0
        TO.add_constraint(p.constraints, TO.LinearConstraint(p.n, p.m, A, [4.0], TO.NegativeOrthant()), (2, N - 1))
    return p


def terms(cls, fourth, error_state=False, B=8, N=31):
    """R3 / E2: two-sided position bounds on knots 2..N and the goal at N (3 AL rows on the position entries: the term slots exactly full),
    the control box; `fourth`: one more upper position bound on knots 2..N-1 (4 rows)"""
    cons = TO.ConstraintList(13, 4, N)
    TO.add_constraint(cons, _pos_bound(lower=(-0.6, -0.3, 0.4)), (2, N))
    _box(cons, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    if fourth:
        TO.add_constraint(cons, _pos_bound(upper=(2.2, 2.5, 2.3)), (2, N - 1))
    return _quad(cls, TO.Objective(_qcost(), _qcost(terminal=True), N), cons, B, N, seed=26, error_state=error_state)


def packed_rows(cls, bound_rows, B=6, N=21):
    """R4: a Bound with `bound_rows` (15 or 16) rows -- the control box and velocity bounds -- on knots 1..N-1 and seven 16-row
    LinearConstraints on knots 2..N-1 (127 / 128 rows at one knot, at most 2 AL terms per z entry)"""
    x_max, x_min = np.full(13, np.inf), np.full(13, -np.inf)
    x_max[7:11], x_min[7:11] = 3.0, -3.0                     # 8 rows + 8 of the control box = 16
    if bound_rows == 15:
        x_min[10] = -np.inf
    cons = TO.ConstraintList(13, 4, N)                        # (8 constraints: the most a problem takes)
    TO.add_constraint(cons, TO.BoundConstraint(13, 4, x_min=x_min, x_max=x_max, u_min=np.zeros(4), u_max=np.full(4, 10.0)), (1, N - 1))
    r = np.random.default_rng(27)
    for _ in range(7):
        A = r.standard_normal((16, 13))
        TO.add_constraint(cons, TO.LinearConstraint(13, 4, A, np.full(16, 40.0), TO.NegativeOrthant()), (2, N - 1))
    return _quad(cls, TO.Objective(_qcost(), _qcost(terminal=True), N), cons, B, N, seed=28)


def dense_knot(cls, dense, B=8, N=31):
    """R5: diagonal costs everywhere, or one dense QuadraticCost (off-diagonal Q, an x-u cross term) on knot 12"""
    stage = _qcost()
    per = [stage] * (N - 1)
    if dense:
        Q = 0.1 * np.eye(13) + 0.002 * (np.ones((13, 13)) - np.eye(13)); R = 0.01 * np.eye(4); H = 0.001 * np.ones((4, 13))
        per[11] = TO.QuadraticCost(Q, R, H=H, q=-Q @ QXF - H.T @ HOVER, r=-R @ HOVER - H @ QXF, c=0.5 * QXF @ Q @ QXF + 0.5 * HOVER @ R @ HOVER + HOVER @ H @ QXF)
    cons = TO.ConstraintList(13, 4, N)
    _box(cons, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    return _quad(cls, TO.Objective(per, _qcost(terminal=True)), cons, B, N, seed=29)


def general_quad(cls, p, B=6, N=21):
    """R6: a goal, a control box and one general constraint of p rows on knots 2..N-1.  p = 16: a SOC NormConstraint over 15 z entries
    (13 states + 2 controls, one row for the norm); p >= 32: p circles far from the flight (a LinearConstraint's A takes fewer rows);
    other p: a LinearConstraint of p rows on the state"""
    cons = TO.ConstraintList(13, 4, N)
    if p == 16:
        TO.add_constraint(cons, TO.NormConstraint(13, 4, 40.0, TO.SecondOrderCone(), list(range(1, 16))), (2, N - 1))
    elif p >= 32:
        TO.add_constraint(cons, TO.CircleConstraint(13, 10.0 + np.arange(p), np.full(p, 10.0), np.full(p, 0.2)), (2, N - 1))
    else:
        A = np.random.default_rng(30).standard_normal((p, 13))
        TO.add_constraint(cons, TO.LinearConstraint(13, 4, A, np.full(p, 40.0), TO.NegativeOrthant()), (2, N - 1))
    _box(cons, N)
    TO.add_constraint(cons, TO.GoalConstraint(QXF), N)
    return _quad(cls, TO.Objective(_qcost(), _qcost(terminal=True), N), cons, B, N, seed=31)


def record_general(cls, general, B=8, N=31):
    """E1: the BASELINE constraints on the error state (the record path), or the same problem plus one general constraint (a cylinder
    around the z axis the flight stays clear of): the materialised expansion and k_riccati_dense_mma"""
    p = TO.problems.quadrotor(B=B, N=N, dt=0.05, error_state=True, cls=cls)
    if general:
        TO.add_constraint(p.constraints, TO.CircleConstraint(13, [5.0], [5.0], [0.5]), (2, N - 1))
    return p


def batch(cls, B, N=21):
    """G1: the BASELINE problem on the error state with B instances"""
    return TO.problems.quadrotor(B=B, N=N, dt=0.05, error_state=True, cls=cls)


# ---- the cases ------------------------------------------------------------------------------------------------------------------

@dataclass
class Case:
    row: str                      # the row of DESIGN.md 4a's table
    side: str
    build: object                 # build(cls, sms, resident) -> problem
    expect: dict                  # the choice this side was built for (a subset of TO.kernel_choice)
    opts: dict = field(default_factory=dict)   # CUDA-side options (backward_kernel)
    big: bool = False             # B sized from the device (R1, G1): a few iterations, no per-instance pipeline
    solve: bool = True            # the solver kernels take it (R6: p = 17 is evaluated only)

    @property
    def name(self):
        return f"{self.row}-{self.side}"


def _c(row, side, fn, expect, **kw):
    return Case(row, side, lambda cls, sms=SMS_H100, resident=RESIDENT_H100: fn(cls), expect, **kw)


CASES = [
    _c("F1", "N512", lambda cls: horizon(cls, 512), dict(linesearch="fast")),
    _c("F1", "N513", lambda cls: horizon(cls, 513), dict(linesearch="generic")),
    _c("F1", "N512_lie", lambda cls: horizon(cls, 512, error_state=True), dict(linesearch="fast", backward="fragment")),
    _c("F1", "N513_lie", lambda cls: horizon(cls, 513, error_state=True), dict(linesearch="generic", backward="fragment")),
    _c("F2", "two", lambda cls: overlap(cls, False), dict(linesearch="fast")),
    _c("F2", "three", lambda cls: overlap(cls, True), dict(linesearch="generic")),
    _c("F3", "p12", lambda cls: rows_per_knot(cls, False), dict(linesearch="fast")),
    _c("F3", "p13", lambda cls: rows_per_knot(cls, True), dict(linesearch="generic")),
    _c("F4", "ncost4", lambda cls: costs(cls, 4), dict(linesearch="fast", cost_cached=True)),
    _c("F4", "ncost5", lambda cls: costs(cls, 5), dict(linesearch="fast", cost_cached=False)),
] + [
    _c("F5", f, (lambda f: lambda cls: compact(cls, f))(f), dict(linesearch="compact" if f == "member" else "fast")) for f in COMPACT_FLIPS
] + [
    Case("R1", f"{mdl}_wave", (lambda mdl: lambda cls, sms=SMS_H100, resident=RESIDENT_H100: small(cls, mdl, SMALL_WAVE * sms))(mdl),
         dict(backward="warp_dfma"), big=True) for mdl in SMALL_MODELS
] + [
    Case("R1", f"{mdl}_wave1", (lambda mdl: lambda cls, sms=SMS_H100, resident=RESIDENT_H100: small(cls, mdl, SMALL_WAVE * sms + 1))(mdl),
         dict(backward="thread"), big=True) for mdl in SMALL_MODELS
] + [
    _c("R2", "diag", lambda cls: small(cls, "cartpole", 8), dict(backward="thread"), opts=dict(backward_kernel=2)),
    _c("R2", "general", lambda cls: small(cls, "cartpole", 8, general=True), dict(backward="warp_dfma", linesearch="generic"),
       opts=dict(backward_kernel=2)),
    _c("R3", "t3", lambda cls: terms(cls, False), dict(backward="warp_mma", fastal=True)),
    _c("R3", "t4", lambda cls: terms(cls, True), dict(backward="warp_mma", fastal=False)),
    _c("R4", "p127", lambda cls: packed_rows(cls, 15), dict(backward="warp_dfma", fastal=True)),
    _c("R4", "p128", lambda cls: packed_rows(cls, 16), dict(backward="warp_dfma", fastal=False)),
    _c("R5", "diag", lambda cls: dense_knot(cls, False), dict(backward="warp_mma")),
    _c("R5", "dense", lambda cls: dense_knot(cls, True), dict(backward="warp_dfma", linesearch="generic")),
    _c("R6", "p16_soc", lambda cls: general_quad(cls, 16), dict(backward="warp_dfma", linesearch="generic")),
    _c("R6", "p17", lambda cls: general_quad(cls, 17), dict(linesearch="generic"), solve=False),
    _c("E1", "records", lambda cls: record_general(cls, False), dict(backward="fragment", late_list=True)),
    _c("E1", "general", lambda cls: record_general(cls, True), dict(backward="dense_mma", late_list=False)),
    _c("E2", "t3", lambda cls: terms(cls, False, error_state=True), dict(backward="fragment", rec_fused=True)),
    _c("E2", "t4", lambda cls: terms(cls, True, error_state=True), dict(backward="fragment", rec_fused=False)),
    Case("G1", "resident", lambda cls, sms=SMS_H100, resident=RESIDENT_H100: batch(cls, resident), dict(backward="fragment"), big=True),
    Case("G1", "resident1", lambda cls, sms=SMS_H100, resident=RESIDENT_H100: batch(cls, resident + 1), dict(backward="fragment"), big=True),
]
BY_NAME = {c.name: c for c in CASES}

# the two sides of every row, and the predicted field that tells them apart (G1 differs in B against the resident count only)
PAIRS = [("F1-N512", "F1-N513", "linesearch"), ("F1-N512_lie", "F1-N513_lie", "linesearch"), ("F2-two", "F2-three", "linesearch"),
         ("F3-p12", "F3-p13", "linesearch"), ("F4-ncost4", "F4-ncost5", "cost_cached")] \
    + [("F5-member", f"F5-{f}", "linesearch") for f in COMPACT_FLIPS[1:]] \
    + [(f"R1-{mdl}_wave", f"R1-{mdl}_wave1", "backward") for mdl in SMALL_MODELS] \
    + [("R2-diag", "R2-general", "backward"), ("R3-t3", "R3-t4", "fastal"), ("R4-p127", "R4-p128", "fastal"), ("R5-diag", "R5-dense", "backward"),
       ("E1-records", "E1-general", "backward"), ("E2-t3", "E2-t4", "rec_fused")]
