"""CPU tests: the oracle against the exact reference (tests/branch_reference.py) on inputs that sit exactly on the branch points of the
AL expansion -- the orthant row at lambda - mu c == 0, the SOC projection at a == s, at the apex and at a == -s -- entry by entry, and the
reference's tie conventions against src/cones.jl read by hand.  The same cases drive tests/test_gpu_branch_points.py."""
import numpy as np
import pytest

import branch_reference as R
import trajopt_b200 as TO
from oracle_binding import OracleProblem, oracle_grad_projection, oracle_hess_projection, oracle_projection


def test_tie_conventions_read_from_cones_jl():
    """cones.jl:141 `J[i,i] = x[i] <= 0 ? 1 : 0`: the orthant row at 0 is active.  cones.jl:151-157 (tested in this order): `a <= -s` is
    below (zero Jacobian), then `a <= s` is in the cone (identity) -- so the boundary a = s > 0 is in, a = -s and the apex are below.
    cones.jl:223-226: the second derivative is zero below and in the cone, the boundary a = s included."""
    assert R.grad_projection(R.NEGATIVE, [0.0, R.EPS, -R.EPS]) == [[1, 0, 0], [0, 0, 0], [0, 0, 1]]
    assert R.projection(R.NEGATIVE, [0.0, R.EPS, -R.EPS]) == [0, 0, -R.EPS]
    assert R.soc_case([3, 4, 5]) == "in" and R.soc_case([0, 0, 0]) == "below" and R.soc_case([-3, -4, -5]) == "below"
    assert R.soc_case([3, 4, -5]) == "below" and R.soc_case([3, 4, 5 - R.EPS]) == "outside"
    assert R.grad_projection(R.SOC, [3, 4, 5]) == [[1, 0, 0], [0, 1, 0], [0, 0, 1]]
    assert R.projection(R.SOC, [3, 4, 5]) == [3, 4, 5]
    for x in ([0, 0, 0], [-3, -4, -5], [3, 4, -5]):
        assert R.grad_projection(R.SOC, x) == R.zeros(3, 3) and R.projection(R.SOC, x) == [0, 0, 0]
        assert R.hess_projection(R.SOC, x, [1, 2, 3]) == R.zeros(3, 3)
    assert R.hess_projection(R.SOC, [3, 4, 5], [1, 2, 3]) == R.zeros(3, 3)
    # outside, s = 0: Pi = (v, a) / 2 and J = [I/2 + 0, v/(2a); v'/(2a), 1/2]  (c = 1/2, cones.jl:163-180)
    J = R.grad_projection(R.SOC, [3, 4, 0])
    assert R.projection(R.SOC, [3, 4, 0]) == [R.Fraction(3, 2), 2, R.Fraction(5, 2)]
    assert J == [[R.Fraction(1, 2), 0, R.Fraction(3, 10)], [0, R.Fraction(1, 2), R.Fraction(2, 5)], [R.Fraction(3, 10), R.Fraction(2, 5), R.Fraction(1, 2)]]


@pytest.mark.parametrize("p", [2, 3, 4, 7])
def test_cone_operators_match_the_reference(p):
    """oracle projection / Jacobian / second derivative at the SOC's branch points and around them, and the orthant at 0 and one step off"""
    pts = R.soc_points(p)
    X = np.array([x for x, _, _ in pts]); Bv = np.array([b for _, b, _ in pts])
    assert [R.soc_case(x) for x in X] == [c for _, _, c in pts]
    P, rc0 = oracle_projection(TO.SecondOrderCone(), X)
    J, rc1 = oracle_grad_projection(TO.SecondOrderCone(), X)
    H, rc2 = oracle_hess_projection(TO.SecondOrderCone(), X, Bv)
    assert rc0 == rc1 == rc2 == 0
    for i, (x, b, case) in enumerate(pts):
        R.assert_entrywise(P[i], R.projection(R.SOC, x), f"projection {case} {x}")
        R.assert_entrywise(J[i], R.grad_projection(R.SOC, x), f"Jacobian {case} {x}")
        # outside the cone the formulas divide by a: their zeros come out of cancellations, measured against the point's largest entry
        Href = R.hess_projection(R.SOC, x, b)
        floor = 0.0 if case != "outside" else float(max(abs(v) for row in Href for v in row))
        R.assert_entrywise(H[i], Href, f"second derivative {case} {x}", ulps=16, floor=floor)
    xo = np.array([[0.0] * p, [R.EPS] * p, [-R.EPS] * p, [0.0, -R.EPS] * (p // 2) + [R.EPS] * (p % 2)])
    Jo, rc = oracle_grad_projection(TO.NegativeOrthant(), xo)
    assert rc == 0
    for i, x in enumerate(xo):
        R.assert_entrywise(Jo[i], R.grad_projection(R.NEGATIVE, x), f"orthant Jacobian {x}")


CASES = {
    "quadrotor_error_state": lambda: R.quadrotor_case(),
    "quadrotor_full_state": lambda: R.quadrotor_case(error_state=False),
    "quadrotor_extra_box": lambda: R.quadrotor_case(extra_box=True),
    "quadrotor_full_state_extra_box": lambda: R.quadrotor_case(error_state=False, extra_box=True),
    "quadrotor_quat_goal": lambda: R.quadrotor_case(quat_goal=True),
    "cartpole": lambda: R.small_case("cartpole"),
    "double_integrator": lambda: R.small_case("double_integrator"),
    "double_integrator_soc": lambda: R.soc_case_problem(),
}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_expansion_at_ties(name):
    """the oracle's AL expansion, merit and violation on the tie inputs equal the exact reference entry by entry; one exact step to the
    other side of every tie moves the expansion by at least mu on some entry (so an expansion on the wrong side cannot pass)"""
    case = CASES[name]()
    o = case.build(OracleProblem, TO)
    merit, viol, G, H = case.reference()
    g, Hh = TO.al_expansion(o)
    R.assert_entrywise(g, G, "gradient"); R.assert_entrywise(Hh, H, "Hessian")
    R.assert_entrywise(TO.merit(o), merit, "merit", ulps=8 * case.N)
    R.assert_entrywise(TO.max_violation(o), viol, "max violation")
    if case.error_state:
        ge, He = TO.error_expansion(o)
        Ge, HHe = case.error_reference()
        R.assert_entrywise(ge, Ge, "error-state gradient"); R.assert_entrywise(He, HHe, "error-state Hessian")
    o.close()
    moved = case.build(OracleProblem, TO, eps=R.EPS)
    _, Hm = TO.al_expansion(moved)
    Href = np.vectorize(float)(np.asarray(H, dtype=object))
    assert np.max(np.abs(Hm - Href)) >= min(c.mu for c in case.cons), "moving the ties did not change the Hessian by a penalty"
    moved.close()


def test_oracle_per_instance_data_at_ties():
    """the per-instance Bound case, one oracle per instance with that instance's data as the constraint's own"""
    case = R.quadrotor_case(inst_data=True)
    merit, viol, G, H = case.reference()
    for b in range(case.B):
        o = case.build(OracleProblem, TO, instance=b)
        g, Hh = TO.al_expansion(o)
        R.assert_entrywise(g[0], G[b], f"instance {b} gradient"); R.assert_entrywise(Hh[0], H[b], f"instance {b} Hessian")
        R.assert_entrywise(TO.merit(o), merit[b:b + 1], f"instance {b} merit", ulps=8 * case.N)
        o.close()
