"""CPU side of the kernel-selection cases (tests/dispatch_cases.py): each pair of problems straddles its threshold in the restated
predicates, each side is the problem it says it is, and the oracle builds and runs both sides (rollout plus one iteration).  The GPU
side (tests/test_gpu_dispatch_boundaries.py) checks that the library lands each side where the restatement says."""
import numpy as np
import pytest

import dispatch_cases as D
import trajopt_b200 as TO
from oracle_binding import OracleProblem

# the oracle runs the R1 / G1 batches (B ~ 16 x 132) at their smallest horizon here; their shape-side is checked through `features` below
SMALL_B = dict(sms=2, resident=40)


def _build(case, cls=OracleProblem, **kw):
    return case.build(cls, **kw) if kw else case.build(cls)


@pytest.mark.parametrize("a,b,fld", D.PAIRS, ids=[p[0].split("-")[0] + ":" + p[1].split("-")[1] for p in D.PAIRS])
def test_pair_straddles_its_threshold(a, b, fld):
    ca, cb = D.BY_NAME[a], D.BY_NAME[b]
    pa, pb = _build(ca), _build(cb)
    sa, sb = D.predicted(pa, **ca.opts), D.predicted(pb, **cb.opts)
    assert sa[fld] != sb[fld], (a, b, fld, sa[fld])
    for case, s in ((ca, sa), (cb, sb)):
        for k, v in case.expect.items():
            assert s[k] == v, f"{case.name}: restated {k} = {s[k]}, the case was built for {v}"
    fa, fb = D.features(pa), D.features(pb)
    row = ca.row
    if row == "F1":
        assert (fa["N"], fb["N"]) == (D.FWD_MAX_N, D.FWD_MAX_N + 1)
    elif row == "F2":
        assert (fa["max_cons_knot"], fb["max_cons_knot"]) == (2, 3)
    elif row == "F3":
        assert (fa["max_p_knot"], fb["max_p_knot"]) == (2 * (fa["n"] + fa["m"]), 2 * (fa["n"] + fa["m"]) + 1)
    elif row == "F4":
        assert (fa["ncost"], fb["ncost"]) == (D.FWD_MAX_COST, D.FWD_MAX_COST + 1)
    elif row == "F5":
        assert fa["fwd_compact"] and not fb["fwd_compact"]
    elif row in ("R3", "E2"):
        assert (fa["max_terms_per_z"], fb["max_terms_per_z"]) == (D.MAXT, D.MAXT + 1)
    elif row == "R4":
        assert (fa["max_p_knot"], fb["max_p_knot"]) == (D.MAXP_KNOT_PACKED - 1, D.MAXP_KNOT_PACKED)
        assert max(fa["max_terms_per_z"], fb["max_terms_per_z"]) <= D.MAXT
    elif row == "R2":
        assert fa["all_diag_con"] and not fb["all_diag_con"]
    elif row == "R5":
        assert fa["all_diag_cost"] and not fb["all_diag_cost"]
    elif row == "E1":
        assert fa["compact"] and not fb["compact"] and fb["lie"]
    pa.close(); pb.close()


@pytest.mark.parametrize("row", ["R1", "G1"])
def test_batch_thresholds(row):
    """R1: B = 16 SMs is the warp kernel, one more instance the thread kernel; G1: B = the resident warps fills the first wave of
    k_riccati_frag exactly, one more instance is pulled from the queue after it (restated at small device sizes)"""
    sms, res = SMALL_B["sms"], SMALL_B["resident"]
    for case in D.CASES:
        if case.row != row:
            continue
        p = case.build(OracleProblem, sms=sms, resident=res)
        full = case.side.endswith("1")
        if row == "R1":
            assert p.B == D.SMALL_WAVE * sms + (1 if full else 0)
            assert D.predicted(p, sms=sms)["backward"] == ("thread" if full else "warp_dfma")
            assert D.predicted(p, sms=D.SMS_H100)["backward"] == "warp_dfma"
        else:
            assert p.B == res + (1 if full else 0)
            assert D.predicted(p)["backward"] == "fragment"
        p.close()


@pytest.mark.parametrize("name", sorted(D.BY_NAME))
def test_oracle_runs_both_sides(name):
    """rollout, cost, the constraints, then one iteration (expand, backward, forward) on the oracle; R1 / G1 at small batches"""
    case = D.BY_NAME[name]
    o = case.build(OracleProblem, **SMALL_B) if case.big else case.build(OracleProblem)
    TO.rollout(o)
    assert np.all(np.isfinite(TO.states(o))) and np.all(np.isfinite(TO.cost(o)))
    for i in range(len(o.constraints)):
        assert np.all(np.isfinite(TO.evaluate_constraints(o, i)))
    assert D.solver_accepts(o) == case.solve
    TO.expand(o)
    TO.backward(o)
    J, alpha = TO.forward(o)
    assert np.all(np.isfinite(J)) and np.all(alpha >= 0)
    o.close()


@pytest.mark.parametrize("p,solver,create", [(16, True, True), (17, False, True), (32, False, True), (33, False, False)])
def test_general_row_limits(p, solver, create):
    """R6 restated: up to 16 rows of a general constraint in the solver kernels, 32 in to_create (the GPU test checks the refusals)"""
    o = D.general_quad(OracleProblem, p)
    assert o.constraints[0].p == p
    assert (D.solver_accepts(o), D.create_accepts(o)) == (solver, create)
    o.close()
