"""CPU check of the ALGORITHM of the record cost-expansion kernel k_expansion_rec16b (rollout.cu): its NumPy restatement
(tests/costexp_emulator.py: term table, 16-knot blocks, activity masks, multiplier pointers, attitude projection, physical order) against the
oracle's dense error-state expansion (Altro error_expansion! restated in oracle/oracle.hpp) on trajectories with active and inactive AL rows."""
import numpy as np
import pytest

import record_configs as rc
import trajopt_b200 as TO
from costexp_emulator import block_images, build_term_table, image_from_dense
from oracle_binding import OracleProblem

P = TO.problems


def _problem(B, N, state_bounds):
    model = TO.Quadrotor(); n, m = 13, 4
    xf = np.array([0, 0, 2, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0])
    obj = TO.LQRObjective(np.full(n, 0.1), np.full(m, 0.01), np.full(n, 100.0), xf, N)
    cons = TO.ConstraintList(n, m, N)
    kw = {}
    if state_bounds:
        x_max = np.full(n, np.inf); x_min = np.full(n, -np.inf)
        x_max[:3] = 2.5; x_min[:3] = -0.5; x_max[7:10] = 1.0; x_min[7:10] = -1.0; x_max[12] = 0.3
        kw = dict(x_min=x_min, x_max=x_max)
    bnd = TO.BoundConstraint(n, m, u_min=np.zeros(4), u_max=np.full(4, 10.0), **kw)
    goal = TO.GoalConstraint(xf)
    TO.add_constraint(cons, bnd, (1, N - 1))
    TO.add_constraint(cons, goal, N)
    r = np.random.default_rng(11)
    x0 = np.broadcast_to(np.array([1, 2, 1, 1, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]), (B, n)).copy(); x0[:, :3] += r.uniform(-1, 1, (B, 3))
    prob = OracleProblem(model, obj, x0, 0.05 * (N - 1), xf=xf, constraints=cons, error_state=True)
    TO.initial_controls(prob, model.hover_control()[None, None, :] + 0.3 * r.standard_normal((B, N - 1, m)))
    return prob, [(bnd, 1, N - 1), (goal, N, N)], xf


@pytest.mark.parametrize("N,state_bounds", [(101, False), (33, True), (16, True), (7, False)])
def test_blocked_cost_expansion_algorithm_matches_the_oracle(N, state_bounds):
    B = 3
    prob, cons, xf = _problem(B, N, state_bounds)
    TO.rollout(prob)
    TO.ilqr_step(prob, 2)
    TO.al_update(prob)                        # non-zero multipliers, penalty 10
    TO.ilqr_step(prob, 1)
    mus = [10.0, 10.0]
    table, offsets, lam_len = build_term_table(cons, mus)
    X, U = TO.states(prob), TO.controls(prob)
    lam = np.zeros((B, lam_len))
    for ci, (c, first, last) in enumerate(cons):
        lam[:, offsets[ci]:offsets[ci] + (last - first + 1) * c.p] = TO.multipliers(prob, c).reshape(B, -1)
    assert np.max(np.abs(lam)) > 0
    Q, R, Qf = np.full(13, 0.1), np.full(4, 0.01), np.full(13, 100.0)
    uf = np.zeros(4)
    costs = [(Q, -Q * xf, R, -R * uf), (Qf, -Qf * xf, R, -R * uf)]
    cost_of_knot = [0] * (N - 1) + [1]
    g_ref, H_ref = TO.error_expansion(prob)
    worst = 0.0
    active = 0
    for b in range(B):
        img = block_images(X[b], U[b], lam[b], table, cost_of_knot, costs, N)
        for k in range(N):
            ref, rest = image_from_dense(g_ref[b, k], H_ref[b, k])
            assert rest < 1e-12, "the expansion of this problem class is diagonal outside the attitude block"
            if k == N - 1:
                ref[[0, 2, 4, 6]] = 0.0; ref[[16, 18, 20, 22]] = 0.0           # no controls at the terminal knot (the kernel writes zeros)
            scale = max(1.0, float(np.max(np.abs(ref))))
            worst = max(worst, float(np.max(np.abs(img[k] - ref))) / scale)
            active += int(np.any(np.abs(np.diag(H_ref[b, k])[12:] - R) > 1e-9))
    assert worst < 1e-12, f"max rel difference {worst:.3e}"
    assert active > 0, "no Bound row was active: the test would not see the AL terms"


def _emulator_vs_oracle(prob):
    """the emulator's images of every knot of `prob` (term table and cost table built from its own description, its current penalties and
    multipliers) against the oracle's dense error-state expansion -> (max relative difference, max |attitude off-diagonal| / block scale)"""
    cons, cost_of_knot, costs = rc.term_inputs(prob)
    table, offsets, lam_len = build_term_table(cons, [TO.penalty(prob, i) for i in range(len(cons))])
    X, U = TO.states(prob), TO.controls(prob)
    B, N = X.shape[:2]
    lam = np.zeros((B, lam_len))
    for ci, (c, first, last) in enumerate(cons):
        lam[:, offsets[ci]:offsets[ci] + (last - first + 1) * c.p] = TO.multipliers(prob, ci).reshape(B, -1)
    g_ref, H_ref = TO.error_expansion(prob)
    worst = offdiag = 0.0
    for b in range(B):
        img = block_images(X[b], U[b], lam[b], table, cost_of_knot, costs, N)
        for k in range(N):
            ref, rest = image_from_dense(g_ref[b, k], H_ref[b, k])
            assert rest < 1e-12
            if k == N - 1:
                ref[[0, 2, 4, 6, 16, 18, 20, 22]] = 0.0
            worst = max(worst, float(np.max(np.abs(img[k] - ref))) / max(1.0, float(np.max(np.abs(ref)))))
            Hb = ref[32:44].reshape(3, 4)[:, :3]
            offdiag = max(offdiag, float(np.max(np.abs(Hb - np.diag(np.diag(Hb))))) / float(np.max(np.abs(np.diag(Hb)))))
    return worst, offdiag


def _natural_iterate(prob):
    TO.rollout(prob)
    TO.ilqr_step(prob, 1); TO.al_update(prob); TO.ilqr_step(prob, 1)
    for i, mu in enumerate((3.7, 11.0, 0.6, 2.3)[:len(prob.constraints)]):     # a distinct penalty per constraint
        TO.set_penalty(prob, i, mu)


@pytest.mark.parametrize("name", ["quat_weights", "state_bounds", "midblock_ranges", "zigzag"])
def test_blocked_cost_expansion_algorithm_on_the_record_configurations(name):
    """the emulated algorithm on the inputs the BASELINE problems never produce (tests/record_configs.py): non-uniform quaternion weights
    (attitude off-diagonals), inequality rows on every state lane, knot ranges that start / end inside 16-knot blocks, one cost per knot"""
    prob = P.quadrotor_zigzag(cls=OracleProblem) if name == "zigzag" else getattr(rc, name)(OracleProblem)
    _natural_iterate(prob)
    worst, offdiag = _emulator_vs_oracle(prob)
    assert worst < 1e-12, f"max rel difference {worst:.3e}"
    if name == "quat_weights":
        assert offdiag > 1e-3, "the attitude block stayed diagonal"
    prob.close()


def test_blocked_cost_expansion_algorithm_on_a_tracking_objective():
    """one cost per knot, re-targeted by update_trajectory and moved by shift_trajectory (MPC), on the error state"""
    prob, Xref, Uref = rc.tracking(OracleProblem)
    for start in (1, 4):
        if start > 1:
            TO.shift_trajectory(prob, 3)
            TO.update_trajectory(prob, Xref, Uref, start)
            TO.rollout(prob)
        _natural_iterate(prob)
        worst, _ = _emulator_vs_oracle(prob)
        assert worst < 1e-12, f"start {start}: max rel difference {worst:.3e}"
    prob.close()
