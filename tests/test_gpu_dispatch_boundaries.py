"""Every shape-driven kernel choice, one step either side of its threshold (tests/dispatch_cases.py, DESIGN.md 4a):

  * the landing test: `TO.kernel_choice` reports the choice the case was built for, and the choice the restated predicates give;
  * against the oracle (parity_util.triple / match_algebra): one kernel application at KERNEL_RTOL, the gains of one expansion + backward
    pass at GAIN_TOL, and the line search, three iterations, an AL update and one more iteration within the divergence of the oracle's
    twin -- on both drivers (overlapped side stream and serial) where the problem's path overlaps;
  * per-instance tables: goals and model parameters g[b % 3] / p[b % 3] reproduce three shared batches bit for bit (the INST kernels).

R1 and G1 size their batches from the device: 16 x the SM count (riccati_small.cu), and the k_riccati_frag warps the occupancy API fits
(`kernel_choice(...)["resident"]`)."""
import functools
import os

import numpy as np
import pytest

import dispatch_cases as D
import trajopt_b200 as TO
from oracle_binding import OracleProblem
from parity_util import GAIN_TOL, check, decisions_agree, triple
from test_gpu_instance_params import G, _compare_pipeline, _model_of, _param_sets, _with_model

pytestmark = pytest.mark.gpu

KERNEL_RTOL = 1e-10      # test_gpu_parity.py: one kernel against the oracle
NAMES = sorted(D.BY_NAME)


@functools.lru_cache(None)
def device_sizes():
    """(SM count, k_riccati_frag warps resident at once) of the device; small stand-ins when the oracle stands in for the library"""
    if TO.Problem is OracleProblem:          # tests/dryrun_gpu_tests_on_oracle.py
        return 2, 40
    import torch
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    p = TO.problems.quadrotor(B=2, N=11, dt=0.05, error_state=True)
    resident = TO.kernel_choice(p)["resident"]
    p.close()
    assert resident > 0
    return sms, resident


def _needs_the_library():
    """the library's own limits and per-instance tables (to_set_model_params, to_set_goal_states) have no oracle counterpart: skipped when
    the oracle stands in for the library"""
    if TO.Problem is OracleProblem:
        pytest.skip("needs the CUDA library (the oracle has no counterpart)")


def _builder(case):
    sms, resident = device_sizes()
    return lambda cls: case.build(cls, sms=sms, resident=resident)


def close(a, b, rtol, what):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(1.0, float(np.max(np.abs(b)))) if b.size else 1.0
    err = float(np.max(np.abs(a - b))) if b.size else 0.0
    assert np.all(np.isfinite(a)) or not np.all(np.isfinite(b)), f"{what}: non-finite GPU result"
    assert err <= rtol * scale, f"{what}: max abs err {err:.3e} > {rtol:.0e} * {scale:.3e}"
    return err / scale


@pytest.mark.parametrize("name", NAMES)
def test_lands_on_its_side(name):
    case = D.BY_NAME[name]
    sms, resident = device_sizes()
    g = _builder(case)(TO.Problem)
    if case.opts:
        TO.set_options(g, **case.opts)
    got = TO.kernel_choice(g)
    print(f"\n{name}: B={g.B} N={g.N} SMs={sms} resident={resident} choice={got}")
    for k, v in case.expect.items():
        assert got[k] == v, f"{name}: {k} = {got[k]}, the case was built for {v}"
    for k, v in D.predicted(g, sms=sms, **case.opts).items():
        assert got[k] == v, f"{name}: {k} = {got[k]}, the restated predicates give {v}"
    assert not got["inst_forward"] and not got["inst_backward"]
    if case.row == "G1":
        assert got["resident"] == resident and g.B == resident + (1 if case.side.endswith("1") else 0)
    if case.row == "R1":
        assert g.B == D.SMALL_WAVE * sms + (1 if case.side.endswith("1") else 0)
    g.close()


def _overlaps(case):
    """the overlapped side stream runs on the full-state and record paths; the materialised error-state path keeps every kernel on the main
    stream.  R1 / G1 (batches sized from the device) run one driver."""
    return not case.big and case.expect.get("backward") not in ("dense_mma", "dense_dfma")


DRIVERS = [(n, "overlap") for n in NAMES] + [(n, "serial") for n in NAMES if _overlaps(D.BY_NAME[n])]


@pytest.mark.parametrize("name,driver", DRIVERS, ids=[f"{n}-{d}" for n, d in DRIVERS])
def test_against_the_oracle(name, driver, monkeypatch):
    case = D.BY_NAME[name]
    if driver == "serial":
        monkeypatch.setenv("TO_NO_OVERLAP", "1")     # read by to_create
    g, o, t = triple(_builder(case), case.opts)
    worst = {}
    for p in (g, o, t):
        TO.rollout(p)
    worst["X"] = close(TO.states(g), TO.states(o), KERNEL_RTOL, "rollout X")
    worst["cost"] = close(TO.cost(g), TO.cost(o), KERNEL_RTOL, "cost")
    worst["cost_knots"] = close(TO.cost_knots(g), TO.cost_knots(o), KERNEL_RTOL, "cost knots")
    worst["grad"] = close(TO.cost_gradient(g), TO.cost_gradient(o), KERNEL_RTOL, "cost gradient")
    worst["hess"] = close(TO.cost_hessian(g), TO.cost_hessian(o), KERNEL_RTOL, "cost hessian")
    for i in range(len(g.constraints)):
        worst[f"c{i}"] = close(TO.evaluate_constraints(g, i), TO.evaluate_constraints(o, i), KERNEL_RTOL, f"constraint {i} values")
        worst[f"J{i}"] = close(TO.constraint_jacobians(g, i), TO.constraint_jacobians(o, i), KERNEL_RTOL, f"constraint {i} jacobians")
    worst["merit"] = close(TO.merit(g), TO.merit(o), KERNEL_RTOL, "merit")
    worst["viol"] = close(TO.max_violation(g), TO.max_violation(o), KERNEL_RTOL, "max violation")
    (gg, gh), (og, oh) = TO.al_expansion(g), TO.al_expansion(o)
    worst["al"] = max(close(gg, og, KERNEL_RTOL, "AL gradient"), close(gh, oh, KERNEL_RTOL, "AL hessian"))
    for p in (g, o, t):
        TO.expand(p)
    worst["AB"] = close(TO.dynamics_jacobians(g), TO.dynamics_jacobians(o), KERNEL_RTOL, "[A B]")
    if not case.solve:       # R6, p = 17: evaluated, and refused by the solver kernels (test_general_row_limits)
        print(f"\n{name}: worst gpu-vs-oracle " + " ".join(f"{k} {v:.1e}" for k, v in worst.items()))
        for p in (g, o, t):
            p.close()
        return
    sg, so, st_ = TO.backward(g), TO.backward(o), TO.backward(t)
    assert np.array_equal(sg, so)
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    worst["K"] = close(Kg, Ko, GAIN_TOL, "K"); worst["d"] = close(dg, do, GAIN_TOL, "d")
    worst["dV"] = close(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"], GAIN_TOL, "dV")
    (Jg, ag), (Jo, ao), (Jt, at) = TO.forward(g), TO.forward(o), TO.forward(t)
    ok = decisions_agree("accepted step sizes", ag, ao, at)
    worst["J fwd"] = check("J after forward pass", Jg, Jo, Jt, 1e-10, ok)[0]
    worst["X fwd"] = check("X after forward pass", TO.states(g), TO.states(o), TO.states(t), 1e-10, ok)[0]
    for p in (g, o, t):
        TO.ilqr_step(p, 3)
        TO.al_update(p)
        TO.ilqr_step(p, 1)
    sg, so, st_ = TO.solver_state(g), TO.solver_state(o), TO.solver_state(t)
    live = np.abs(so["dV"][:, 0]) > 1e-9 * np.maximum(1.0, np.abs(TO.merit(o)))
    dec = live & (so["alpha"] == st_["alpha"]) & (so["bp_status"] == st_["bp_status"]) & (sg["alpha"] == so["alpha"]) & (sg["bp_status"] == so["bp_status"])
    worst["merit it"] = check("merit after the iterations", TO.merit(g), TO.merit(o), TO.merit(t), 1e-8, dec, outliers=0.05)[0]
    worst["X it"] = check("X after the iterations", TO.states(g), TO.states(o), TO.states(t), 1e-8, dec, outliers=0.05)[0]
    worst["U it"] = check("U after the iterations", TO.controls(g), TO.controls(o), TO.controls(t), 1e-8, dec, outliers=0.05)[0]
    worst["rho"] = check("rho", sg["rho"], so["rho"], st_["rho"], 1e-12, dec, outliers=0.05)[0]
    for k in ("alpha", "ls_iters", "bp_status"):
        decisions_agree(k, sg[k], so[k], st_[k], live, allow=0.05)
    for i in range(len(g.constraints)):
        worst[f"lambda{i}"] = check(f"multipliers {i}", TO.multipliers(g, i), TO.multipliers(o, i), TO.multipliers(t, i), 1e-8, dec, outliers=0.05)[0]
        assert TO.penalty(g, i) == TO.penalty(o, i)
    print(f"\n{name} [{driver}]: worst gpu-vs-oracle " + " ".join(f"{k} {v:.1e}" for k, v in worst.items()))
    for p in (g, o, t):
        p.close()


def test_general_row_limits():
    """R6: 17 rows of a general constraint are evaluated (test_against_the_oracle) but refused by to_backward / to_ilqr_step with TO_ESTATE;
    to_create takes 32 rows and refuses 33 with TO_EINVAL"""
    _needs_the_library()
    g = D.general_quad(TO.Problem, 17)
    TO.rollout(g); TO.expand(g)
    for call in (lambda: TO.backward(g), lambda: TO.ilqr_step(g, 1)):
        with pytest.raises(TO.TrajOptError, match="at most 16 rows"):
            call()
    assert g._lib.to_backward(g._h, None) == TO.capi.TO_ESTATE and g._lib.to_ilqr_step(g._h, 1) == TO.capi.TO_ESTATE
    g.close()
    g = D.general_quad(TO.Problem, 32)
    TO.rollout(g)
    assert TO.evaluate_constraints(g, 0).shape[-1] == 32
    g.close()
    with pytest.raises(TO.ArgumentError, match="bad size"):
        D.general_quad(TO.Problem, 33)


INST = [n for n in NAMES if D.BY_NAME[n].solve and not D.BY_NAME[n].big]


@pytest.mark.parametrize("name", INST)
def test_instance_tables_equal_shared_batches(name):
    """goals g[b % 3] and model parameters p[b % 3] on one batch against three shared batches: the INST variant of each kernel the case
    lands on computes, row for row, what the shared kernel computes"""
    _needs_the_library()
    case = D.BY_NAME[name]
    build = _builder(case)
    per = build(TO.Problem)
    if case.opts:
        TO.set_options(per, **case.opts)
    sets = _param_sets(per.model)
    rng = np.random.default_rng(7)
    goals = []
    for _ in range(G):
        gl = np.array(per.xf, dtype=float); gl[:2] += rng.uniform(-0.3, 0.3, 2); goals.append(gl)
    TO.set_model_params(per, np.stack([sets[b % G] for b in range(per.B)]))
    TO.set_goal_state(per, np.stack([goals[b % G] for b in range(per.B)]))
    choice = TO.kernel_choice(per)
    assert choice["inst_forward"] and choice["inst_backward"]
    for k, v in case.expect.items():
        assert choice[k] == v, f"{name}: {k} = {choice[k]} with per-instance tables"
    shared = []
    for j in range(G):
        s = build(_with_model(_model_of(per.model, sets[j])))
        if case.opts:
            TO.set_options(s, **case.opts)
        TO.set_goal_state(s, goals[j])
        shared.append(s)
    _compare_pipeline(per, shared, name)
    for p in [per] + shared:
        p.close()
