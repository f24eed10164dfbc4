"""The integration rule of a problem (``Problem(..., integration)``, include/trajopt_b200.h to_set_integration) on the host: argument checks
and round trips, the reference's own test of the keyword (test/problems_tests.jl:87-88) restated, the oracle's four rules (tests/oracle_rules.cpp)
against NumPy restatements of the rules, the restatements and the oracle on the double integrator (where every rule but Euler is exact), and
the declarations of the new entry points.  No GPU needed."""
import os
import re

import numpy as np
import pytest

import trajopt_b200 as TO
from integration_rules import RULES, RulesOracleProblem, double_integrator_step_errors, jacobian_fd, model_step, rollout, step
from oracle_binding import oracle_dynamics

P = TO.problems
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rule_codes_and_forms():
    """the codes of to_integration, from a rule type, an instance (``RD.RK3(model)``) or a name"""
    for name, code in (("Euler", 1), ("RK2", 2), ("RK3", 3), ("RK4", 4)):
        rule = getattr(TO, name)
        assert rule.code == code
        assert TO.api._integration_code(rule) == code
        assert TO.api._integration_code(rule(TO.Cartpole())) == code
        assert TO.api._integration_code(name) == code
        assert rule() == rule(TO.Cartpole()) and rule() != TO.RK4() or name == "RK4"


@pytest.mark.parametrize("rule", ["ImplicitMidpoint", "HermiteSimpson", "rk4", "RK5", "", 4, 3.0, None, object, TO.api._Integration])
def test_unknown_and_implicit_rules_are_refused(rule):
    with pytest.raises(TO.ArgumentError, match="integration rule"):
        TO.api._integration_code(rule)


def test_refused_before_the_handle_exists():
    """Problem(...; integration = RD.ImplicitMidpoint): ArgumentError, and no handle is opened"""
    opened = []

    class Probe(RulesOracleProblem):
        def _open(self):
            opened.append(1)
            super()._open()

    with pytest.raises(TO.ArgumentError, match="ImplicitMidpoint"):
        P.cartpole(B=1, N=11, cls=Probe, integration="ImplicitMidpoint")
    assert not opened


def test_problems_tests_integration_keyword():
    """test/problems_tests.jl:87-88: ``Problem(model, obj, x0, tf; integration = RD.Euler(model))`` keeps the rule,
    ``RD.integration(prob.model[1]) isa RD.Euler``; the default is RK4.  Then round trips with RK3."""
    e = P.cartpole(B=2, N=11, cls=RulesOracleProblem, integration=TO.Euler(TO.Cartpole()))
    assert isinstance(TO.integration(e), TO.Euler)
    p = P.cartpole(B=2, N=11, cls=RulesOracleProblem)
    assert isinstance(TO.integration(p), TO.RK4) and p._integration == 4
    q = P.cartpole(B=2, N=11, cls=RulesOracleProblem, integration=TO.RK3)
    assert isinstance(TO.integration(q), TO.RK3) and TO.integration(q) == TO.RK3()
    # copy(prob) carries the rule; an override replaces it
    assert isinstance(TO.integration(TO.copy_problem(q)), TO.RK3)
    assert isinstance(TO.integration(TO.copy_problem(q, integration="RK4")), TO.RK4)
    TO.set_integration(q, "RK4")
    assert isinstance(TO.integration(q), TO.RK4)
    with pytest.raises(TO.ArgumentError):
        TO.set_integration(q, "HermiteSimpson")
    assert isinstance(TO.integration(q), TO.RK4)
    with pytest.raises(TO.TrajOptError, match="unknown integration rule 7"):
        q._raw_call("to_set_integration", 7)
    assert isinstance(TO.integration(q), TO.RK4)
    for x in (e, p, q):
        x.close()


def test_oracle_rules_against_numpy():
    """The oracle's rollout and [A B] with each rule against the NumPy restatements, on the Cartpole and the Quadrotor; the Jacobians against
    central differences of the restatement."""
    for build, tol in ((lambda cls, **kw: P.cartpole(B=2, N=21, cls=cls, **kw), 1e-12),
                       (lambda cls, **kw: P.quadrotor(B=2, N=11, cls=cls, **kw), 1e-12)):
        for name in sorted(RULES):
            p = build(RulesOracleProblem, integration=name)
            TO.rollout(p)
            X, U, t = TO.states(p), TO.controls(p), TO.gettimes(p)
            stp = model_step(p.model, name)
            for b in range(p.B):
                ref = rollout(stp, p.x0[b], U[b], np.diff(t))
                assert np.allclose(X[b], ref, rtol=tol, atol=tol), (name, b)
            TO.expand(p)
            AB = TO.dynamics_jacobians(p)
            for b in range(p.B):
                # central differences lose digits in proportion to the state: knots of a rollout that has grown large are left out
                for k in [k for k in (0, p.N // 2, p.N - 2) if np.abs(X[b, k:k + 2]).max() < 100.0]:
                    fd = jacobian_fd(stp, X[b, k], U[b, k], t[k + 1] - t[k])
                    assert np.allclose(AB[b, k], fd, rtol=1e-6, atol=1e-7), (name, b, k)
            p.close()


@pytest.mark.parametrize("rule", sorted(RULES))
def test_restatements_on_the_cartpole_and_quadrotor_jacobians(rule):
    """every restated rule: its order of accuracy on the Cartpole (halving h divides the one-step error by about 2^(order+1)) and a
    central-difference Jacobian that is consistent with the step on the Quadrotor"""
    order = {"Euler": 1, "RK2": 2, "RK3": 3, "RK4": 4}[rule]
    cp = TO.Cartpole()
    x, u = np.array([0.1, 0.5, -0.2, 0.3]), np.array([0.7])
    def fine(h, sub=256):             # the reference: RK4 with 256 substeps
        y = x.copy()
        for _ in range(sub):
            y = step(lambda a, b: oracle_dynamics(cp, a, b), y, u, h / sub, "RK4")
        return y
    e1 = np.linalg.norm(step(lambda a, b: oracle_dynamics(cp, a, b), x, u, 0.08, rule) - fine(0.08))
    e2 = np.linalg.norm(step(lambda a, b: oracle_dynamics(cp, a, b), x, u, 0.04, rule) - fine(0.04))
    assert abs(np.log2(e1 / e2) - (order + 1)) < 0.6, (rule, e1, e2)
    q = TO.Quadrotor()
    stp = model_step(q, rule)
    xq = np.array([1.0, 2.0, 1.0, 0.9, 0.1, -0.2, 0.3, 0.2, -0.1, 0.3, 0.4, -0.5, 0.2])
    xq[3:7] /= np.linalg.norm(xq[3:7])
    uq = np.array([1.3, 1.2, 1.4, 1.1])
    J = jacobian_fd(stp, xq, uq, 0.05)
    dz = 1e-7 * np.linspace(-1.0, 1.0, 17)
    lin = stp(xq, uq, 0.05) + J @ dz
    assert np.allclose(stp(xq + dz[:13], uq + dz[13:], 0.05), lin, rtol=0, atol=1e-12)
    # the closed-form position / velocity columns (rollout.cu SeedList): d r+/d r = I, d r+/d v = h I, d v+/d v = I for every rule
    assert np.allclose(J[:, 0:3], np.eye(13)[:, 0:3], atol=1e-8)
    assert np.allclose(J[0:3, 7:10], 0.05 * np.eye(3), atol=1e-8) and np.allclose(J[7:10, 7:10], np.eye(3), atol=1e-8)


@pytest.mark.parametrize("rule", sorted(RULES))
def test_double_integrator_exactness(rule):
    """x'' = u/m with a constant u: RK2, RK3 and RK4 integrate it exactly; Euler is off by exactly h^2 a / 2 in position and exact in velocity"""
    di = TO.DoubleIntegrator(2)
    a = np.array([0.8, -1.7]) / di.params[0]
    x, u, h = np.array([0.3, -0.4, 1.1, 0.2]), np.array([0.8, -1.7]), 0.1
    xn = model_step(di, rule)(x, u, h)
    exact = np.concatenate([x[:2] + h * x[2:] + 0.5 * h * h * a, x[2:] + h * a])
    if rule == "Euler":
        assert np.allclose(exact[:2] - xn[:2], 0.5 * h * h * a, rtol=1e-12, atol=1e-15)
        assert np.allclose(xn[2:], exact[2:], rtol=1e-14, atol=1e-15)
    else:
        assert np.allclose(xn, exact, rtol=1e-14, atol=1e-15)


@pytest.mark.parametrize("rule", sorted(RULES))
def test_oracle_double_integrator_exactness(rule):
    """the oracle's rollout of the double integrator (1-D and 2-D): every step of RK2, RK3 and RK4 is the exact solution under constant u;
    Euler's is off by h^2 a / 2 in position and exact in velocity"""
    for dim, N in ((1, 51), (2, 21)):
        p = P.double_integrator(B=3, N=N, dim=dim, cls=RulesOracleProblem, integration=rule)
        TO.initial_controls(p, np.random.default_rng(3).standard_normal((3, N - 1, dim)))
        TO.rollout(p)
        X, U, h = TO.states(p), TO.controls(p), np.diff(TO.gettimes(p))
        for b in range(3):
            dr, dv = double_integrator_step_errors(X[b], U[b], h, p.model.params[0])
            scale = max(1.0, np.abs(X[b]).max())
            if rule == "Euler":
                dr = dr + 0.5 * (h * h)[:, None] * U[b] / p.model.params[0]
            assert np.abs(dr).max() < 1e-13 * scale and np.abs(dv).max() < 1e-13 * scale, (rule, dim, b)
        p.close()


def test_declarations():
    """the entry points in the ctypes binding, the header (with the codes of orc_set_integrator) and the Julia shim"""
    assert {"to_set_integration", "to_get_integration"} <= set(TO.capi.EXPORTED_SYMBOLS)
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert "enum to_integration { TO_EULER = 1, TO_RK2 = 2, TO_RK3 = 3, TO_RK4 = 4 };" in hdr
    assert re.search(r"int to_set_integration\(to_handle\* h, int32_t rule\);", hdr)
    assert re.search(r"int to_get_integration\(const to_handle\* h, int32_t\* rule\);", hdr)
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert "integration=RD.integration(TO.get_model(prob)[1])" in jl and ":to_set_integration" in jl and ":to_get_integration" in jl
    for t, c in (("Euler", 1), ("RK2", 2), ("RK3", 3), ("RK4", 4)):
        assert f"integration_code(::RD.{t}) = Int32({c})" in jl
