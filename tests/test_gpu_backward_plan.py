"""The backward pass each problem and `backward_kernel` option runs, and what follows from it (csrc/riccati.cu backward_plan).

For every path, after a rollout and an expansion:
  * `TO.kernel_choice` reports the kernel the case lands on, and what the restated predicates (tests/dispatch_cases.py) give;
  * `TO.backward_algebra` is 1 and `TO.expansion_records` answers exactly on the record path;
  * one `TO.backward` launches the kernels its plan needs: the record expansion and k_riccati_frag on the record path; on the
    shared-memory error-state path the ABe export (record problems), the compact or the materialised expansion, the error-state
    Jacobians (without a Lie-group state) and the kernel; one kernel otherwise;
  * `to_algorithmic_bytes` counts the bytes of the expansion that backward pass reads, restated below from SURVEY.md 8(d).

Cartpole's batches are sized from the device, as in tests/test_gpu_dispatch_boundaries.py: 16 x the SM count is the last batch the
automatic choice leaves on the warp kernel."""
import ctypes as C

import pytest

import dispatch_cases as D
import trajopt_b200 as TO
from oracle_binding import OracleProblem
from test_gpu_dispatch_boundaries import device_sizes
from test_gpu_instance_params import _quickstart
from trajopt_b200 import problems

pytestmark = pytest.mark.gpu

EC_LEN = 40      # common.cuh TO_EC_LEN: doubles of a knot's compact expansion


def _quad_es(sms):
    return problems.quadrotor(B=8, N=31, dt=0.05, error_state=True)


def _cartpole(extra):
    return lambda sms: D.small(TO.Problem, "cartpole", D.SMALL_WAVE * sms + extra)


CASES = [   # (name, build(SM count) -> problem, backward_kernel, the kernel it lands on)
    *[("quadrotor_error_state", _quad_es, o, k) for o, k in ((0, "fragment"), (1, "fragment"), (2, "fragment"), (3, "dense_dfma"),
                                                           (5, "dense_mma"))],
    ("records_descriptor_walk", lambda sms: D.terms(TO.Problem, True, error_state=True), 0, "fragment"),
    *[("quadrotor_lie", lambda sms: problems.quadrotor_lie(B=8, N=31), o, k) for o, k in ((0, "dense_mma"), (3, "dense_dfma"))],
    *[("quadrotor_full_state", lambda sms: problems.quadrotor(B=8, N=31, dt=0.05), o, "warp_mma") for o in (0, 1, 2, 3)],
    *[("cartpole_wave", _cartpole(0), o, k) for o, k in ((0, "warp_dfma"), (1, "warp_dfma"), (2, "thread"))],
    *[("cartpole_wave1", _cartpole(1), o, k) for o, k in ((0, "thread"), (1, "warp_dfma"), (2, "thread"))],
    ("double_integrator_quickstart", lambda sms: _quickstart(8), 0, "warp_dfma"),
]
IDS = [f"{name}-bk{o}" for name, _, o, _ in CASES]


def _expansion(f, kernel, option):
    """where the backward pass reads its cost + AL expansion"""
    if kernel == "fragment":
        return "records"
    if f["dense_riccati"]:
        return "compact" if f["compact"] and option != 3 else "materialised"
    return "in_kernel"


def _launches(f, expansion):
    """kernels one to_backward launches"""
    if expansion == "records":
        return 2
    if expansion in ("compact", "materialised"):
        return int(f["compact"]) + (1 if expansion == "compact" else 2) + int(not f["lie"]) + 1
    return 1


def _bytes(prob, f, expansion):
    """to_algorithmic_bytes (E, R, F) restated: SURVEY.md 8(d), with R counting the expansion the backward pass reads"""
    n, m, N, ne, w = prob.n, prob.m, prob.N, prob.ne, 8
    XU, AB, KD = (n + m) * N, n * (n + m) * (N - 1), m * (ne + 1) * (N - 1)
    L = sum((b - a + 1) * c.p for (a, b), c in zip(prob.constraints.inds, prob.constraints.constraints))
    dense = f["dense_riccati"]
    HES = ((ne + m) ** 2 + (ne + m)) * N if dense else 0
    ABe = ne * (ne + m) * (N - 1) if dense else 0
    HESF = ((n + m) ** 2 + (n + m)) * N
    R = {"records": ABe + XU + KD + L,
         "compact": XU + L + 2 * EC_LEN * N + ABe + KD,
         "materialised": XU + L + 2 * HESF + 2 * HES + (0 if f["lie"] else AB + ABe) + ABe + KD,
         "in_kernel": AB + XU + KD + L}[expansion]
    E = XU + ABe if f["lie"] else XU + AB
    return E * w, R * w, (2 * XU + KD + L) * w + 8


@pytest.mark.parametrize("name,build,option,kernel", CASES, ids=IDS)
def test_backward_plan(name, build, option, kernel):
    if TO.Problem is OracleProblem:          # tests/dryrun_gpu_tests_on_oracle.py: the oracle has no kernel choice or launch count
        pytest.skip("needs the CUDA library (the oracle has no counterpart)")
    sms, _ = device_sizes()
    g = build(sms)
    TO.set_options(g, backward_kernel=option)
    TO.rollout(g)
    TO.expand(g)
    got = TO.kernel_choice(g)
    assert got["backward"] == kernel, f"{name}: backward = {got['backward']}, the case was built for {kernel}"
    for k, v in D.predicted(g, backward_kernel=option, sms=sms).items():
        assert got[k] == v, f"{name}: {k} = {got[k]}, the restated predicates give {v}"
    on_records = kernel == "fragment"
    assert TO.backward_algebra(g) == (1 if on_records else 0)

    f = D.features(g)
    expansion = _expansion(f, kernel, option)
    before = g._lib.to_launch_count(g._h)
    TO.backward(g)
    assert g._lib.to_launch_count(g._h) - before == _launches(f, expansion), f"{name}: kernels launched by one backward pass"
    if on_records:
        assert TO.expansion_records(g).shape == (g.B, g.N, 48)
    else:
        with pytest.raises(TO.TrajOptError, match="not on the record path"):
            TO.expansion_records(g)

    E, R, F = C.c_int64(), C.c_int64(), C.c_int64()
    assert g._lib.to_algorithmic_bytes(g._h, C.byref(E), C.byref(R), C.byref(F)) == 0
    assert (E.value, R.value, F.value) == _bytes(g, f, expansion), f"{name}: algorithmic bytes with the {expansion} expansion"
    g.close()
