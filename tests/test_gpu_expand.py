"""The error-state dynamics expansion of the record path (rollout.cu k_expand_lie_rec) must write the same [A_e B_e] blocks, bit for bit, as
the expansion into P.ABe (k_expand_lie, closed-form columns from k_trivial_columns) -- at the benchmark size and at sizes with partial knot
blocks.  Both compute every seed column with expand_lie_column and the closed-form columns with the same formula.  The second problem is
the first plus a CircleConstraint: the constraint leaves the dynamics alone and takes the problem out of the compact class."""
import numpy as np
import pytest

import trajopt_b200 as TO

pytestmark = pytest.mark.gpu


def test_record_dynamics_expansion_equals_the_abe_expansion():
    for B, N in ((4096, 101), (1, 2), (3, 5), (33, 2), (2, 64), (5, 23)):
        rec = TO.problems.quadrotor(B=B, N=N, error_state=True)
        cons = TO.ConstraintList(13, 4, N)
        for inds, c in zip(rec.constraints.inds, rec.constraints.constraints):
            TO.add_constraint(cons, c, inds)
        TO.add_constraint(cons, TO.CircleConstraint(13, [5.0], [5.0], [0.5]), (1, N))
        # a new problem, not add_constraint on rec's list: rebuilding a live handle re-derives the time steps from its knot times
        full = TO.Problem(rec.model, rec.obj, rec.x0, 5.0, xf=rec.xf, constraints=cons, error_state=True)
        TO.initial_controls(full, TO.controls(rec))
        assert TO.backward_algebra(rec) == 1 and TO.backward_algebra(full) != 1, (B, N)
        for p in (rec, full):
            TO.rollout(p)
            TO.expand(p)
        assert np.array_equal(TO.states(rec), TO.states(full)), (B, N)
        a, b = TO.error_dynamics(rec), TO.error_dynamics(full)
        assert np.all(np.isfinite(a)), (B, N)
        assert np.array_equal(a, b), f"B = {B}, N = {N}: max |record - ABe| = {np.max(np.abs(a - b)):.3e}"
        # the closed-form columns (positions, velocities): 1 on the diagonal
        assert np.all(a[..., [0, 1, 2, 6, 7, 8], [0, 1, 2, 6, 7, 8]] == 1.0), (B, N)
        rec.close(); full.close()
