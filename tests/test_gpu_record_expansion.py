"""GPU tests (`-m gpu`) of the cost + AL expansion that the record path's Riccati kernel reads: doubles [192, 240) of every knot's record,
written by rollout.cu k_expansion_rec16b (term table) or riccati_frag.cu k_expansion_rec (more than 3 Goal / Bound rows on one z entry, or
N >= 4095), read back with expansion_records (to_get_expansion_records).

Method: the CUDA problem is iterated to a natural iterate (non-zero multipliers, active rows); its trajectory and multipliers are copied
into the oracle and both sides get the same distinct penalties, so both expand IDENTICAL inputs -- no closed-loop amplification, no twin
budget.  The records are compared with the image (costexp_emulator.image_from_dense) of the oracle's dense error-state expansion, then
the gains of the backward pass with the oracle's.  Every configuration asserts that it reaches what it is there for (tests/record_configs.py)."""
import numpy as np
import pytest

import record_configs as rc
import trajopt_b200 as TO
from costexp_emulator import image_from_dense
from oracle_binding import OracleProblem, match_algebra
from parity_util import GAIN_TOL, check, decisions_agree, triple

pytestmark = pytest.mark.gpu
K = TO.capi
P = TO.problems

# the emulated algorithm agrees with the oracle to ~1e-15 (test_costexp_emulator.py); the kernels' FMA contraction adds a few ulps
REC_RTOL = 1e-11
KERNEL_RTOL = 1e-10
PENALTIES = (3.7, 11.0, 0.6, 2.3)
CTRL = [0, 2, 4, 6]                          # physical slots of u_0..u_3 (frag_layout.cuh)


def close(a, b, rtol, what):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(1.0, float(np.max(np.abs(b))))
    err = float(np.max(np.abs(a - b)))
    assert np.all(np.isfinite(a)), f"{what}: non-finite GPU result"
    assert err <= rtol * scale, f"{what}: max abs err {err:.3e} > {rtol:.0e} * {scale:.3e}"


def natural_iterate(g):
    TO.rollout(g)
    TO.ilqr_step(g, 1); TO.al_update(g); TO.ilqr_step(g, 1)


def set_penalties(p, mus=PENALTIES):
    for i in range(len(p.constraints)):
        TO.set_penalty(p, i, mus[i])


def copy_iterate(g, o):
    """the CUDA problem's trajectory and multipliers into the oracle"""
    TO.initial_controls(o, TO.controls(g)); TO.initial_states(o, TO.states(g))
    for i in range(len(g.constraints)):
        TO.set_multipliers(o, i, TO.multipliers(g, i))


def reset_regularisation(*probs):
    """rho = drho = 0 on every instance (to_set_options resets them when bp_reg_initial changes): the oracle is a fresh problem"""
    for p in probs:
        TO.set_options(p, bp_reg_initial=1e-8); TO.set_options(p, bp_reg_initial=0.0)


def active_rows(o):
    """[B, N, n+m]: the AL rows' share of the full-state Hessian diagonal (oracle), 0 where no row of that entry is active"""
    _, Hal = TO.al_expansion(o)
    d = np.diagonal(Hal, axis1=-2, axis2=-1) - np.diagonal(TO.cost_hessian(o), axis1=-2, axis2=-1)
    return np.where(np.abs(d) > 1e-12, d, 0.0)


def records_vs_oracle(g, o, exact_symmetry=False):
    """expand + backward on the CUDA side; its records against the oracle's error-state expansion of the same inputs, and the records'
    invariants -> (max relative error, max |attitude off-diagonal| / max |attitude diagonal| of the records).
    Symmetry of the attitude block: k_expansion_rec writes each off-diagonal once into both triangles (`exact_symmetry`: bit for bit);
    the term-table kernels compute Hb[a][b] = sum_r (G_a[r] h_r) G_b[r] in lane / step a and Hb[b][a] = sum_r (G_b[r] h_r) G_a[r] in
    b, two roundings of the same sum.  Each is within gamma_5 sum_r |G_a[r] h_r G_b[r]| <= 5 u max_r |h_r| |q|^2 of it (one product,
    four FMAs; |G_a| = |G_b| = |q|), so they may differ by 10 u max|h_q| |q|^2 -- the bound below, rounded up to 12 u."""
    TO.expand(g); TO.backward(g)
    R = TO.expansion_records(g)
    ge, He = TO.error_expansion(o)
    B, N = g.B, g.N
    assert R.shape == (B, N, 48) and np.all(np.isfinite(R))
    assert not np.any(R[:, -1, CTRL]) and not np.any(R[:, -1, [16 + c for c in CTRL]]), "the terminal knot has no controls"
    worst = 0.0
    for b in range(B):
        for k in range(N):
            ref, rest = image_from_dense(ge[b, k], He[b, k])
            assert rest < 1e-12, "the oracle's expansion of this class is diagonal outside the attitude block"
            if k == N - 1:
                ref[CTRL] = 0.0; ref[[16 + c for c in CTRL]] = 0.0
            worst = max(worst, float(np.max(np.abs(R[b, k] - ref))) / max(1.0, float(np.max(np.abs(ref)))))
    assert worst <= REC_RTOL, f"records vs oracle: max rel err {worst:.3e}"
    Hb, hd = R[..., 32:].reshape(B, N, 4, 4), R[..., 16:32]
    asym = np.abs(Hb - np.swapaxes(Hb, -1, -2)).max(axis=(-1, -2))
    if exact_symmetry:
        assert not np.any(asym), "Hb is not symmetric"
    else:
        _, Hal = TO.al_expansion(o)
        hq = np.abs(np.diagonal(Hal, axis1=-2, axis2=-1)[..., 3:7]).max(axis=-1)
        bound = 12 * np.finfo(float).eps / 2 * hq * np.sum(TO.states(o)[..., 3:7] ** 2, axis=-1)
        assert np.all(asym <= bound), f"Hb asymmetric beyond rounding: {np.max(asym / bound):.2f} x the bound"
        print(f"Hb asymmetry up to {np.max(asym / bound):.2f} x the rounding bound")
    for a in range(3):
        assert np.array_equal(Hb[..., a, a], hd[..., 8 + 2 * a]), f"Hb[{a}][{a}] != hd[{8 + 2 * a}]"
        assert not np.any(Hb[..., a, 3]), f"Hb[{a}][3] != 0"
    assert np.array_equal(Hb[..., 3, 3], hd[..., 14]), "Hb[3][3] != hd[14]"
    att = Hb[..., :3, :3]
    off = np.abs(att - np.einsum("...ii->...i", att)[..., None] * np.eye(3))
    return worst, float(np.max(off.max(axis=(-1, -2)) / np.abs(np.einsum("...ii->...i", att)).max(axis=-1)))


def gains_vs_oracle(g, o):
    """backward pass of both from rho = 0 (the CUDA problem expanded by the caller)"""
    TO.expand(o)
    reset_regularisation(g, o)
    sg, so = TO.backward(g), TO.backward(o)
    assert np.array_equal(sg, so), (sg, so)
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    close(Kg, Ko, GAIN_TOL, "K"); close(dg, do, GAIN_TOL, "d")
    close(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"], GAIN_TOL, "dV")


def pair(build, iterate=natural_iterate):
    """(CUDA problem at its iterate, oracle problem with the same trajectory, multipliers and penalties)"""
    g = build(TO.Problem)
    o = match_algebra(g, build(OracleProblem))
    assert TO.backward_algebra(g) == 1, "not on the record path"
    iterate(g)
    copy_iterate(g, o)
    for p in (g, o):
        set_penalties(p)
    return g, o


def run(build, iterate=natural_iterate, exact_symmetry=False):
    g, o = pair(build, iterate)
    worst, offdiag = records_vs_oracle(g, o, exact_symmetry)
    act = active_rows(o)
    gains_vs_oracle(g, o)
    print(f"records vs oracle: max rel err {worst:.2e}; attitude off-diagonal / diagonal up to {offdiag:.2e}")
    g.close(); o.close()
    return worst, offdiag, act


def test_records_before_any_backward_pass_and_off_the_record_path():
    g = P.quadrotor(B=2, N=11, dt=0.05, error_state=True)
    TO.rollout(g); TO.expand(g)
    with pytest.raises(TO.TrajOptError, match="before any backward"):
        TO.expansion_records(g)
    TO.backward(g)
    assert TO.expansion_records(g).shape == (2, 11, 48)
    TO.set_options(g, backward_kernel=5)        # shared-memory kernel on the compact expansion: the records are not read
    with pytest.raises(TO.TrajOptError, match="not on the record path"):
        TO.expansion_records(g)
    g.close()
    f = P.quadrotor(B=2, N=11, dt=0.05)
    TO.rollout(f); TO.expand(f); TO.backward(f)
    with pytest.raises(TO.TrajOptError, match="not on the record path"):
        TO.expansion_records(f)
    f.close()


def test_baseline():
    """the benchmarked problem (B = 33 of it)"""
    _, _, act = run(lambda cls: P.quadrotor(B=33, N=101, error_state=True, cls=cls))
    assert np.any(act[:, :-1, 13:]), "no control row active"


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("N", [2, 3, 15, 16, 17, 33])
def test_edge_sizes(B, N):
    """partial 16-knot blocks, a block of one knot, the terminal knot alone in its block (N = 17, 33)"""
    run(lambda cls: P.quadrotor(B=B, N=N, dt=0.05, error_state=True, cls=cls))


def test_quat_weights():
    _, offdiag, _ = run(rc.quat_weights)
    assert offdiag > 1e-3, f"attitude off-diagonals only {offdiag:.1e} of the diagonal"


def test_state_bounds():
    _, _, act = run(rc.state_bounds)
    stage = act[:, 1:-1]
    for name, js in (("position", [0, 1, 2]), ("quaternion", [3, 4, 5, 6]), ("velocity", [7, 8, 9])):
        assert np.any(stage[..., js]), f"no active inequality row on the {name} entries"
    assert np.any(stage[..., 3]), "q_w >= 0.9 never active"
    goal_mu = PENALTIES[2]
    assert np.any(act[:, -1, :13] > goal_mu + 1e-9), "no state bound row active at the terminal knot beside the goal"


def test_midblock_ranges():
    _, _, act = run(rc.midblock_ranges)
    (a0, a1), (b0, _), kg = rc.MIDBLOCK["A"], rc.MIDBLOCK["B"], rc.MIDBLOCK["G"]
    assert np.any(act[:, 32:a1, :13]), "bound A has no active state row in its last (partial) block"
    assert np.any(act[:, b0 - 1:48, 7:10]), "bound B has no active row in its first (partial) block"
    assert np.all(act[:, kg - 1, [3, 4, 5, 6, 10, 11, 12]] > 0), "the goal at knot 50 does not act"


def test_per_knot_costs_zigzag():
    """examples/Quadrotor.ipynb: waypoint costs at knots 33 (a block's first knot), 66 (inside a block) and the terminal cost"""
    run(lambda cls: P.quadrotor_zigzag(cls=cls, error_state=True))


def test_per_knot_costs_tracking_mpc():
    """TrackingObjective (a cost per knot) re-targeted by update_trajectory and moved by shift_trajectory, on the error state"""
    built = {}

    def build(cls):
        built[cls], Xref, Uref = rc.tracking(cls)
        built["ref"] = (Xref, Uref)
        return built[cls]
    g, o = pair(build)
    for start in (1, 4):
        if start > 1:
            for p in (g, o):
                TO.shift_trajectory(p, 3)
                TO.update_trajectory(p, *built["ref"], start)
            natural_iterate(g)
            copy_iterate(g, o)
            for p in (g, o):
                set_penalties(p)
        worst, _ = records_vs_oracle(g, o)
        gains_vs_oracle(g, o)
        print(f"start {start}: records vs oracle max rel err {worst:.2e}")
    g.close(); o.close()


def test_four_terms_fallback():
    """5 rows on the position entries: k_expansion_rec (descriptor walk) writes the records"""
    assert rc.max_terms_per_z(rc.four_terms(OracleProblem)) > 3
    _, offdiag, act = run(rc.four_terms, exact_symmetry=True)
    assert np.any(act[:, 2:-1, :3]), "no bound row active on the position"
    assert offdiag > 1e-3, f"attitude off-diagonals only {offdiag:.1e} of the diagonal"


def _hand_multipliers(g):
    """a rollout of hover + noise; multipliers set by hand: bound rows of both signs around the activity threshold, the goal's at random"""
    TO.rollout(g)
    r = np.random.default_rng(8)
    for i, c in enumerate(g.constraints):
        shape = TO.multipliers(g, i).shape
        TO.set_multipliers(g, i, r.normal(0, 2, shape) if isinstance(c, TO.GoalConstraint) else r.uniform(-12.0, 1.0, shape))


@pytest.mark.parametrize("N", [4094, 4095])
def test_twelve_bit_knot_field(N):
    """N = 4094: the last horizon of the term table (k_expansion_rec16b); N = 4095: k_expansion_rec"""
    _, _, act = run(lambda cls: rc.long_horizon(cls, N), iterate=_hand_multipliers, exact_symmetry=(N == 4095))
    assert np.any(act[:, :-1, 13:]), "no control row active"


# ---- split vs unsplit -------------------------------------------------------------------------------------------------------------------
# the benchmarked problem at the benchmark size and smaller, sizes with partial 6- and 16-knot blocks, and Bound rows on states and controls
SPLIT = {
    "baseline": lambda cls: P.quadrotor(B=256, N=101, error_state=True, cls=cls),
    "state_bounds": lambda cls: rc.state_bounds(cls, B=256),
    "quadrotor_4096x101": lambda cls: P.quadrotor(B=4096, N=101, error_state=True, cls=cls),
    "quadrotor_37x101": lambda cls: P.quadrotor(B=37, N=101, error_state=True, cls=cls),
    "quadrotor_5x23": lambda cls: P.quadrotor(B=5, N=23, error_state=True, cls=cls),
    "calm_37x101": lambda cls: P.quadrotor(B=37, N=101, error_state=True, u_noise=0.01, cls=cls),
    "calm_5x33": lambda cls: P.quadrotor(B=5, N=33, error_state=True, u_noise=0.01, cls=cls),
    "calm_64x16": lambda cls: P.quadrotor(B=64, N=16, error_state=True, u_noise=0.01, cls=cls),
    "bounded_6x40": lambda cls: rc.bounded(cls, B=6, N=40),
}


@pytest.mark.parametrize("name", list(SPLIT))
def test_split_expansion_equals_unsplit(name):
    """an iteration that follows one whose line search needed the later passes expands the instances accepted by pass 1 (mode 1) and the
    late ones (mode 2, through the late list) separately; a fresh expand + backward of the same trajectory must give the same records and
    gains, bit for bit.  a and b take the same iterations (an AL update after the third) until b's last one leaves late instances; then a
    takes one more."""
    a, b = SPLIT[name](TO.Problem), SPLIT[name](TO.Problem)
    for p in (a, b):
        TO.rollout(p)
    for it in range(10):
        TO.ilqr_step(a, 1); TO.ilqr_step(b, 1)
        if np.any(TO.solver_state(b)["ls_iters"] > 4):
            break
        if it == 2:
            TO.al_update(a); TO.al_update(b)
    assert np.any(TO.solver_state(b)["ls_iters"] > 4), "no instance needed the later line-search passes: no iteration was split"
    TO.ilqr_step(a, 1)
    TO.expand(b); TO.backward(b)
    Ra, Rb = TO.expansion_records(a), TO.expansion_records(b)
    assert np.array_equal(Ra, Rb), f"max |split - unsplit| = {np.max(np.abs(Ra - Rb)):.3e}"
    (Ka, da), (Kb, db) = TO.gains(a), TO.gains(b)
    assert np.array_equal(Ka, Kb) and np.array_equal(da, db)
    a.close(); b.close()


@pytest.mark.parametrize("name", [k for k in SPLIT if k not in ("baseline", "state_bounds", "quadrotor_4096x101")])
def test_split_configurations_against_the_oracle(name):
    """the records of the configurations above against the oracle's expansion"""
    g, o = pair(SPLIT[name])
    worst, _ = records_vs_oracle(g, o)
    print(f"records vs oracle: max rel err {worst:.2e}")
    g.close(); o.close()


# ---- setters on the record path --------------------------------------------------------------------------------------------------------
def _setters(g):
    """(name, action(p)) pairs; each action is applied to both problems with the same arguments"""
    r = np.random.default_rng(9)
    xf2 = rc.XF.copy(); xf2[:3] = (0.3, -0.2, 1.7); xf2[7:10] = (0.05, 0.0, -0.05)
    nref = g.N + 5
    Xref = np.tile(rc.XF, (nref, 1)); Xref[:, 0] = np.linspace(0, 1, nref); Xref[:, 2] = 1.5
    Uref = np.tile(rc.HOVER, (nref, 1)) + 0.1
    lam = [1.5 * TO.multipliers(g, i) + r.normal(0, 0.5, TO.multipliers(g, i).shape) for i in range(len(g.constraints))]
    out = [(f"set_penalty({i})", lambda p, i=i: TO.set_penalty(p, i, 2.0 + 3.0 * i)) for i in range(len(g.constraints))]
    out += [(f"set_multipliers({i})", lambda p, i=i: TO.set_multipliers(p, i, lam[i])) for i in range(len(g.constraints))]
    # the C entry points directly: the mirror API re-creates a handle whose objective it has changed (Problem._ensure_current)
    out += [(f"set_goal_state(objective={ob}, constraint={cn})", lambda p, ob=ob, cn=cn: p._raw_call("to_set_goal_state", K._dp(xf2), ob, cn))
            for ob, cn in ((1, 0), (0, 1), (1, 1))]
    out += [("set_options(penalty_initial)", lambda p: TO.set_options(p, penalty_initial=2.5))]
    out += [("update_trajectory", lambda p: p._raw_call("to_update_trajectory", K._dp(Xref), K._dp(Uref), nref, 3))]
    return out


@pytest.mark.parametrize("error_state", [True, False])
def test_setters_after_an_overlapped_iteration(error_state):
    """each setter right after ilqr_step (its late line-search trials still pending on the side stream), on both sides: merit and violation,
    then (record path) the records against the oracle, and the gains.  Full state: the lane-resident term path of k_riccati, gains only."""
    g = rc.state_bounds(TO.Problem, B=8, error_state=error_state)
    o = match_algebra(g, rc.state_bounds(OracleProblem, B=8, error_state=error_state))
    assert TO.backward_algebra(g) == (1 if error_state else 0)
    TO.rollout(g)
    TO.ilqr_step(g, 1); TO.al_update(g)
    for p in (g, o):
        set_penalties(p)
    for name, action in _setters(g):
        TO.ilqr_step(g, 1)
        action(g)                                  # first call after the step: joins the side stream
        copy_iterate(g, o)
        action(o)
        close(TO.merit(g), TO.merit(o), KERNEL_RTOL, f"{name}: merit")
        close(TO.max_violation(g), TO.max_violation(o), KERNEL_RTOL, f"{name}: max violation")
        if error_state:
            worst, _ = records_vs_oracle(g, o)
            print(f"{name}: records vs oracle max rel err {worst:.2e}")
        else:
            TO.expand(g)
        gains_vs_oracle(g, o)
    g.close(); o.close()


# ---- full-state fallback ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["four_terms", "N4095"])
def test_full_state_descriptor_walk(name):
    """full state beyond the lane-resident term table (5 rows on one entry; N = 4095): k_riccati<FASTAL = false>.  Gains, dV and one
    forward pass against the oracle, with hand-set multipliers and distinct penalties"""
    build = (lambda cls: rc.four_terms(cls, error_state=False)) if name == "four_terms" else (lambda cls: rc.long_horizon(cls, 4095, error_state=False))
    g, o, t = triple(build)
    assert TO.backward_algebra(g) == 0
    _hand_multipliers(g)
    for p in (o, t):
        TO.rollout(p)
        for i in range(len(g.constraints)):
            TO.set_multipliers(p, i, TO.multipliers(g, i))
    for p in (g, o, t):
        set_penalties(p)
        TO.expand(p)
    assert np.any(active_rows(o)[:, :-1]), "no AL row active"
    sg, so = TO.backward(g), TO.backward(o); TO.backward(t)
    assert np.array_equal(sg, so)
    (Kg, dg), (Ko, do) = TO.gains(g), TO.gains(o)
    close(Kg, Ko, GAIN_TOL, "K"); close(dg, do, GAIN_TOL, "d")
    close(TO.solver_state(g)["dV"], TO.solver_state(o)["dV"], GAIN_TOL, "dV")
    (Jg, ag), (Jo, ao), (Jt, at) = TO.forward(g), TO.forward(o), TO.forward(t)
    ok = decisions_agree("accepted step sizes", ag, ao, at)
    check("J after forward pass", Jg, Jo, Jt, 1e-10, ok)
    check("X after forward pass", TO.states(g), TO.states(o), TO.states(t), 1e-10, ok)
    for p in (g, o, t):
        p.close()
