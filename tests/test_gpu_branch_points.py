"""GPU tests (`-m gpu`): every kernel that evaluates an AL branch point or the Quadrotor's motor relu, on inputs exactly at the tie
(tests/branch_reference.py cases: dyadic inputs, power-of-two penalties, Pythagorean SOC vectors -- lambda - mu c and the SOC norm are exact in
any evaluation order, so every correct kernel must take the reference's side).

Each case asserts the backward kernel it lands on, then compares
  * the sweep's al_expansion, merit and max_violation with the exact reference, entry by entry;
  * on the record path, the records with the exact image of the reference's error-state expansion;
  * backward status, K, d and dV with the oracle expanded on the same inputs (GAIN_TOL per knot, identical status) -- on every backward
    kernel, also those whose in-kernel expansion is not exposed;
and proves that it can fail: the oracle with every tie moved by one exact step (2^-20) to the other side of its branch gives gains that differ
from the at-tie gains by at least 10^3 x GAIN_TOL."""
import numpy as np
import pytest

import branch_reference as R
import record_configs as rc
import trajopt_b200 as TO
from costexp_emulator import image_from_dense
from oracle_binding import OracleProblem, match_algebra, oracle_discrete_dynamics
from parity_util import GAIN_TOL
from test_gpu_record_expansion import reset_regularisation

pytestmark = pytest.mark.gpu
CTRL = [0, 2, 4, 6]                          # physical slots of u_0..u_3 in a record (frag_layout.cuh)

CASES = [   # (id, case, backward_kernel option, the kernel it lands on, rec_fused, fastal)
    ("quadrotor_error_state-rec16b", lambda: R.quadrotor_case(), 0, "fragment", True, False),
    ("quadrotor_error_state_extra_box-rec", lambda: R.quadrotor_case(extra_box=True), 0, "fragment", False, False),
    ("quadrotor_error_state-compact_bk5", lambda: R.quadrotor_case(), 5, "dense_mma", False, False),
    ("quadrotor_error_state-materialised_bk3", lambda: R.quadrotor_case(), 3, "dense_dfma", False, False),
    ("quadrotor_quat_goal-materialised", lambda: R.quadrotor_case(quat_goal=True), 0, "dense_mma", False, False),
    ("quadrotor_full_state-fastal", lambda: R.quadrotor_case(error_state=False), 0, "warp_mma", False, True),
    ("quadrotor_full_state-bk3", lambda: R.quadrotor_case(error_state=False), 3, "warp_mma", False, True),
    ("quadrotor_full_state_extra_box-descriptor_walk", lambda: R.quadrotor_case(error_state=False, extra_box=True), 0, "warp_mma", False, False),
    ("cartpole-warp_bk1", lambda: R.small_case("cartpole"), 1, "warp_dfma", False, True),
    ("cartpole-thread_bk2", lambda: R.small_case("cartpole"), 2, "thread", False, False),
    ("double_integrator-warp_bk1", lambda: R.small_case("double_integrator"), 1, "warp_dfma", False, True),
    ("double_integrator-thread_bk2", lambda: R.small_case("double_integrator"), 2, "thread", False, False),
    ("double_integrator_soc-general", lambda: R.soc_case_problem(), 0, "warp_dfma", False, True),
    ("quadrotor_error_state_inst_data-rec16b", lambda: R.quadrotor_case(inst_data=True), 0, "fragment", True, False),
    ("quadrotor_full_state_inst_data-fastal", lambda: R.quadrotor_case(error_state=False, inst_data=True), 0, "warp_mma", False, True),
]


def knot_err(a, b):
    """max over (instance, knot) of |a - b| / max(1, max |b|) of that knot"""
    a, b = np.asarray(a), np.asarray(b)
    ax = tuple(range(2, b.ndim))
    return float(np.max(np.abs(a - b).max(axis=ax) / np.maximum(1.0, np.abs(b).max(axis=ax))))


def oracle_backward(case, g, eps=0.0):
    """(status, K, d, dV) of the oracle on the case's inputs moved by eps, in the arithmetic form of g; one oracle per instance when the case
    has per-instance constraint data"""
    insts = [None] if not case.inst_bounds(0.0) else list(range(case.B))
    out = []
    for b in insts:
        o = match_algebra(g, case.build(OracleProblem, TO, eps=eps, instance=b))
        TO.expand(o)
        reset_regularisation(o)
        s = TO.backward(o)
        K, d = TO.gains(o)
        out.append((s, K, d, TO.solver_state(o)["dV"]))
        o.close()
    return tuple(np.concatenate([r[i] for r in out]) for i in range(4))


@pytest.mark.parametrize("cid,make,option,kernel,rec_fused,fastal", CASES, ids=[c[0] for c in CASES])
def test_branch_points(cid, make, option, kernel, rec_fused, fastal):
    case = make()
    g = case.build(TO.Problem, TO)
    TO.set_options(g, backward_kernel=option)
    TO.expand(g)
    got = TO.kernel_choice(g)
    for what, want in (("backward", kernel), ("rec_fused", rec_fused), ("fastal", fastal)):
        assert got[what] == want, f"{cid}: {what} = {got[what]}, the case was built for {want}"
    if "extra_box" in cid:
        assert rc.max_terms_per_z(g) > 3, "the case does not leave the term table"
    assert TO.backward_algebra(g) == (1 if kernel == "fragment" else 0)

    # the sweep against the exact reference
    merit, viol, G, H = case.reference()
    gs, Hs = TO.al_expansion(g)
    R.assert_entrywise(gs, G, "al_expansion gradient"); R.assert_entrywise(Hs, H, "al_expansion Hessian")
    R.assert_entrywise(TO.merit(g), merit, "merit", ulps=8 * case.N)
    R.assert_entrywise(TO.max_violation(g), viol, "max violation")

    # the backward pass (and on the record path the records it read)
    TO.expand(g)
    reset_regularisation(g)
    sg = TO.backward(g)
    if kernel == "fragment":
        Ge, He = case.error_reference()
        Rg = TO.expansion_records(g)
        for b in range(case.B):
            for k in range(case.N):
                ref, rest = image_from_dense(np.vectorize(float)(np.asarray(Ge[b][k], dtype=object)), np.vectorize(float)(np.asarray(He[b][k], dtype=object)))
                assert rest == 0.0
                if k == case.N - 1:
                    ref[CTRL] = 0.0; ref[[16 + c for c in CTRL]] = 0.0
                R.assert_entrywise(Rg[b, k], ref, f"record of instance {b} knot {k}")
    Kg, dg = TO.gains(g)
    dVg = TO.solver_state(g)["dV"]
    so, Ko, do, dVo = oracle_backward(case, g)
    assert np.array_equal(sg, so), (sg, so)
    assert np.all(sg == 0), f"backward status {sg}"
    for what, a, b in (("K", Kg, Ko), ("d", dg, do), ("dV", dVg[:, None, :], dVo[:, None, :])):
        e = knot_err(a, b)
        assert np.all(np.isfinite(a)) and e <= GAIN_TOL, f"{what}: max rel err per knot {e:.3e} > {GAIN_TOL:.0e}"

    # the case can fail: on the other side of every tie the gains move by >= 1e3 x the tolerance
    _, Km, dm, _ = oracle_backward(case, g, eps=R.EPS)
    moved = max(knot_err(Km, Ko), knot_err(dm, do))
    assert moved >= 1e3 * GAIN_TOL, f"moving the ties changes the gains by only {moved:.2e}"
    print(f"{cid}: gains vs oracle within tolerance; the moved ties change them by {moved:.2e}")
    g.close()


@pytest.mark.parametrize("p", [2, 3, 4, 7])
def test_cone_operators_at_branch_points(p):
    """to_projection / to_grad_projection / to_hess_projection (costcon.cuh cone_*) at the SOC's branch points against the exact reference"""
    pts = R.soc_points(p)
    X = np.array([x for x, _, _ in pts]); Bv = np.array([b for _, b, _ in pts])
    P, J = TO.projection(TO.SecondOrderCone(), X), TO.grad_projection(TO.SecondOrderCone(), X)
    H = TO.hess_projection(TO.SecondOrderCone(), X, Bv)
    for i, (x, b, case) in enumerate(pts):
        R.assert_entrywise(P[i], R.projection(R.SOC, x), f"projection {case} {x}")
        R.assert_entrywise(J[i], R.grad_projection(R.SOC, x), f"Jacobian {case} {x}")
        Href = R.hess_projection(R.SOC, x, b)
        floor = 0.0 if case != "outside" else float(max(abs(v) for row in Href for v in row))
        R.assert_entrywise(H[i], Href, f"second derivative {case} {x}", ulps=16, floor=floor)
    xo = np.array([[0.0] * p, [R.EPS] * p, [-R.EPS] * p])
    Jo = TO.grad_projection(TO.NegativeOrthant(), xo)
    for i, x in enumerate(xo):
        R.assert_entrywise(Jo[i], R.grad_projection(R.NEGATIVE, x), f"orthant Jacobian {x}")


def _motor_problem(cls, error_state, w):
    """full-state / error-state Quadrotor, B = 3, N = 4, dt = 1/16, the case's states at rest (zero rates: no gyroscopic coupling): instance 0 with
    motors (0, 0, 0, 0) (the closed form of the tie), instance 1 with motors (0, w, 0, w) -- some at the tie, the others at w -- and
    instance 2 with every motor at w"""
    case = R.quadrotor_case(error_state=error_state, N=4)
    p = case.build(cls, TO)
    X = case.inputs(0.0)[0]; X[..., 10:13] = 0.0
    U = np.zeros((3, 3, 4)); U[1, :, 1::2] = w; U[2] = w
    TO.initial_states(p, X); TO.initial_controls(p, U)
    return p


@pytest.mark.parametrize("error_state,per_instance", [(False, False), (False, True), (True, False)],
                         ids=["full_state-k_expand", "full_state-per_instance_params", "error_state-error_dynamics"])
def test_motor_tie(error_state, per_instance):
    """max(0, kf w) at w = 0: derivative 0 (SURVEY.md section 7) in k_expand (shared and per-instance parameters) and the error-state
    Jacobians, entry by entry against the oracle; with every motor at 0 the thrust columns vanish (test_oracle_kats.py
    test_relu_tie_convention); at w = 2^-30 they do not"""
    g, o = _motor_problem(TO.Problem, error_state, 3.0), _motor_problem(OracleProblem, error_state, 3.0)
    if per_instance:
        TO.set_model_params(g, [TO.Quadrotor()] * 3)
    for p in (g, o):
        TO.expand(p)
    get = TO.error_dynamics if error_state else TO.dynamics_jacobians
    Ag, Ao = get(g), get(o)
    ne = g.ne
    err = np.abs(Ag - Ao) / np.maximum(np.abs(Ao), 1e-300)
    assert np.all((Ag == Ao) | (err <= 1e-12)), f"Jacobians vs oracle: max rel err per entry {np.max(err[Ag != Ao]):.2e}"
    v, w = (slice(7, 10), slice(10, 12)) if not error_state else (slice(6, 9), slice(9, 11))
    yaw = 12 if not error_state else 11
    assert not np.any(Ag[0][:, v, ne:]) and not np.any(Ag[0][:, w, ne:]), "thrust columns at w = 0 are not zero"
    assert np.all(Ag[0][:, yaw, ne:] != 0), "the motor torque column vanished"
    assert np.all(np.abs(Ag[2][:, v, ne:]).max(axis=1) > 1e-3)
    if not error_state:
        # the left difference quotient (f(x, u) - f(x, u - h e_j)) / h: at w = 0 both sides of the thrust are 0, so it sees the tie's
        # derivative 0 (the right quotient would see kf); loose tolerance, O(h) truncation at the motors at w > 0
        X, U, h = TO.states(g), TO.controls(g), 2.0 ** -20
        for b in range(2):
            f0 = oracle_discrete_dynamics(g.model, X[b, 0], U[b, 0], 1 / 16)
            for j in range(4):
                e = np.zeros(4); e[j] = h
                fd = (f0 - oracle_discrete_dynamics(g.model, X[b, 0], U[b, 0] - e, 1 / 16)) / h
                col = Ag[b, 0, :, ne + j]
                assert np.max(np.abs(col - fd)) <= 1e-4 * max(1.0, np.max(np.abs(col))), f"instance {b} motor {j}: Jacobian column vs left quotient"
    g.close(); o.close()
    m = _motor_problem(OracleProblem, error_state, 3.0)
    TO.initial_controls(m, np.full((3, 3, 4), 2.0 ** -30))
    TO.expand(m)
    assert np.all(np.abs(get(m)[0][:, v, ne:]).max(axis=1) > 1e-3), "one step off the tie the thrust columns stay zero"
    m.close()
