"""CPU tests of the padded size classes of recorded-program problems, (4, 2), (8, 4) and (16, 8): the rule that picks a problem's class
(to_recorded_dims, and the size-class oracle's statement of it, tests/oracle_classes.cpp), that oracle's class checks, Problem's padding onto
the class, the oracle's interpreter on (8, 4) and (16, 8) programs against NumPy and central differences, and the declarations in the header,
the ctypes binding, INTEGRATION.md and the Julia shim."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import trajopt_b200 as TO
from dynamics_programs import model_ops, numpy_jacobian, numpy_step, pad
from recorded_classes import (CLASS_PROGRAMS, ClassesOracleProblem, arm7_model, class_model, load_classes_oracle, padded_closed_form,
                              planar_quadrotor_model, quadrotor_model)

K = TO.capi
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H = 0.1


def expected_class(nx, nu):
    for n, m in ((4, 2), (8, 4), (16, 8)):
        if nx <= n and nu <= m:
            return n, m
    return None


def oracle_rule(nx, nu):
    lib = load_classes_oracle()
    n, m = C.c_int32(), C.c_int32()
    rc = lib.orc_recorded_dims(nx, nu, C.byref(n), C.byref(m))
    return rc, (n.value, m.value)


def test_rule_at_every_dimension():
    """the smallest class holding both dimensions, from the library and from the oracle, at every (nx_max, nu_max) in 1..16 x 0..8"""
    for nx in range(1, 17):
        for nu in range(0, 9):
            want = expected_class(nx, nu)
            assert K.recorded_dims(nx, nu) == want, (nx, nu)
            assert oracle_rule(nx, nu) == (K.TO_OK, want), (nx, nu)


@pytest.mark.parametrize("nx,nu", [(17, 0), (17, 1), (2, 9), (16, 9), (17, 8), (100, 100)])
def test_rule_refuses_past_16_by_8(nx, nu):
    with pytest.raises(TO.DimensionMismatch, match="at most 16 states and 8 controls"):
        K.recorded_dims(nx, nu)
    lib = K.load_library()
    n, m = C.c_int32(-7), C.c_int32(-7)
    assert lib.to_recorded_dims(nx, nu, C.byref(n), C.byref(m)) == K.TO_EDIM and (n.value, m.value) == (-7, -7)
    assert oracle_rule(nx, nu)[0] == K.TO_EDIM


def test_rule_refuses_empty_dimensions_and_null_outputs():
    lib = K.load_library()
    n, m = C.c_int32(), C.c_int32()
    for nx, nu in ((0, 1), (-1, 0), (3, -1)):
        assert lib.to_recorded_dims(nx, nu, C.byref(n), C.byref(m)) == K.TO_EINVAL
        assert oracle_rule(nx, nu)[0] == K.TO_EINVAL
    assert lib.to_recorded_dims(4, 2, None, C.byref(m)) == K.TO_EINVAL
    assert lib.to_recorded_dims(4, 2, C.byref(n), None) == K.TO_EINVAL


# ---- the size-class oracle's orc_create: the class of a spec -----------------------------------------------------------------------------------------------------
def class_spec(model, n, m, N=4, B=2, nx=None, nu=None, dyn=None):
    """a recorded-program spec of N knots stepped by `model`, on the padded layout (n, m)"""
    costs = [dict(kind=K.COST_DIAGONAL, Q=np.ones(n), R=np.ones(m), q=np.zeros(n), r=np.zeros(m), c=0.0),
             dict(kind=K.COST_DIAGONAL, Q=np.ones(n), R=np.ones(m), q=np.zeros(n), r=np.zeros(m), c=0.0, terminal=True)]
    return K.Spec(K.MODEL_EXPR, n, m, N, B, np.full(N - 1, 0.1), costs, [0] * (N - 1) + [1], [], dyn=[dyn or model._spec()],
                  dyn_index=[0] * (N - 1), nx=list(nx or [model.n] * N), nu=list(nu or [model.m] * N))


def orc_create(spec):
    lib = load_classes_oracle()
    h = C.c_void_p()
    rc = lib.orc_create(C.byref(spec.c), C.byref(h))
    msg = lib.orc_last_error(None).decode()
    if h:
        lib.orc_destroy(h)
    return rc, bool(h), msg


@pytest.mark.parametrize("model_fn,cls", [(planar_quadrotor_model, (8, 4)), (quadrotor_model, (16, 8)), (arm7_model, (16, 8))])
def test_oracle_create_takes_only_the_class(model_fn, cls):
    model = model_fn()
    rc, made, msg = orc_create(class_spec(model, *cls))
    assert rc == K.TO_OK and made, msg
    for n, m in ((4, 2), (8, 4), (16, 8), (16, 4), (13, 4), (model.n, model.m)):
        if (n, m) == cls:
            continue
        rc, made, msg = orc_create(class_spec(model, n, m))
        assert rc == K.TO_EDIM and not made, (n, m)
        assert f"run on the padded size class n = {cls[0]}, m = {cls[1]}" in msg, msg


def test_oracle_create_refuses_dimensions_past_the_largest_class():
    model = planar_quadrotor_model()
    rc, made, msg = orc_create(class_spec(model, 16, 8, nx=[17, 6, 6, 6]))
    assert rc == K.TO_EDIM and not made and "at most 16 states and 8 controls per knot, the largest has (17, 2)" in msg
    rc, made, msg = orc_create(class_spec(model, 16, 8, nu=[2, 9, 2, 2]))
    assert rc == K.TO_EDIM and not made and "the largest has (6, 9)" in msg


def test_oracle_create_refuses_models_outside_the_class():
    """n_in / m_in / n_out past the class the knots' dimensions give: the program-size check, before the per-knot checks"""
    model = planar_quadrotor_model()
    bad = "recorded-program model: bad program size or dimensions"
    for field, v in (("n_in", 9), ("m_in", 5), ("n_out", 9)):
        d = dict(model._spec()); d[field] = v
        rc, made, msg = orc_create(class_spec(model, 8, 4, dyn=d))
        assert rc == K.TO_EINVAL and not made and bad in msg, field


# ---- Problem: padding onto the class -----------------------------------------------------------------------------------------------------
def lqr_problem(model, N=5, B=2):
    n, m = model.n, model.m
    obj = TO.LQRObjective(np.ones(n), np.ones(m), np.ones(n), np.zeros(n), N)
    return ClassesOracleProblem(model, obj, np.zeros(n), 1.0, batch=B)


@pytest.mark.parametrize("model_fn,cls", [(planar_quadrotor_model, (8, 4)), (quadrotor_model, (16, 8)), (arm7_model, (16, 8)),
                                          (lambda: TO.AutodiffDynamics(5, 2, lambda x, u: [x[1], x[2], x[3], x[4], u[0] - u[1]]), (8, 4)),
                                          (lambda: TO.AutodiffDynamics(2, 3, lambda x, u: [x[1], u[0] + u[1] + u[2]]), (8, 4))])
def test_problem_takes_the_class(model_fn, cls):
    model = model_fn()
    p = lqr_problem(model)
    assert p.hybrid and (p.n, p.m) == cls and p.nx == [model.n] * p.N and p.nu == [model.m] * p.N
    assert (p.spec.c.n, p.spec.c.m) == cls
    q = ClassesOracleProblem(model, p.obj, p.x0, 1.0)          # x0 on the padded layout, as p.x0 holds it
    assert np.array_equal(q.x0, p.x0)
    with pytest.raises(TO.DimensionMismatch, match="x0 does not match"):
        ClassesOracleProblem(model, p.obj, p.x0 + 1.0, 1.0) if cls[0] != model.n else ClassesOracleProblem(model, p.obj, np.ones(model.n + 1), 1.0)
    p.close(); q.close()


@pytest.mark.parametrize("n,m", [(17, 1), (2, 9)])
def test_problem_refuses_past_16_by_8(n, m):
    model = TO.AutodiffDynamics(n, m, lambda x, u: [x[(i + 1) % n] + u[i % m] for i in range(n)])
    with pytest.raises(TO.DimensionMismatch, match="at most 16 states and 8 controls"):
        lqr_problem(model)


# ---- the oracle's interpreter on (8, 4) and (16, 8) programs -----------------------------------------------------------------------------
def rel_err(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b)), initial=0.0))


def test_the_class_programs_record_every_op_code():
    for name in CLASS_PROGRAMS:
        model = class_model(name)
        assert model_ops(model) == set(range(20)), name
        assert len(model.prog) <= K.EXPR_MAXLEN


@pytest.mark.parametrize("discrete", [False, True], ids=["rk4", "jump_map"])
@pytest.mark.parametrize("name", sorted(CLASS_PROGRAMS) + ["quadrotor", "arm7"])
def test_oracle_interpreter_against_numpy_and_central_differences(name, discrete):
    model = {"quadrotor": quadrotor_model, "arm7": arm7_model}.get(name, lambda: class_model(name))()
    if discrete:
        model = TO.AutodiffDynamics(model.n, model.m, model.fun, discrete=True)
    n, m = model.n, model.m
    cn, cm = K.recorded_dims(n, m)
    B = 16
    r = np.random.default_rng(5)
    x = r.uniform(-1.0, 1.0, (B, n))
    u = r.uniform(-1.0, 1.0, (B, m))
    if name == "quadrotor":
        x[:, 3:7] /= np.linalg.norm(x[:, 3:7], axis=1, keepdims=True)
        u = r.uniform(0.5, 2.0, (B, m))
    if name.startswith("ops"):
        x[:, 0] = np.linspace(-1.0, 1.0, B)
    N = 2
    obj = TO.LQRObjective(np.ones(n), np.ones(m), np.ones(n), np.zeros(n), N)
    p = ClassesOracleProblem(model, obj, np.zeros(n), H, batch=B)
    assert (p.n, p.m) == (cn, cm)
    TO.set_initial_state(p, pad(x, cn))
    TO.initial_controls(p, pad(u, cm)[:, None, :])
    TO.rollout(p); TO.expand(p)
    Xn, AB = TO.states(p)[:, 1], TO.dynamics_jacobians(p)[:, 0]
    ref = np.stack([numpy_step(model, x[b], u[b], H) for b in range(B)])
    assert rel_err(Xn[:, :n], ref) < 1e-13
    assert np.all(Xn[:, n:] == 0.0)
    fd = np.stack([numpy_jacobian(model, x[b], u[b], H) for b in range(B)])
    got = np.concatenate([AB[:, :n, :n], AB[:, :n, cn:cn + m]], axis=-1)
    assert np.allclose(got, fd, rtol=1e-6, atol=1e-7), f"max |[A B] - central differences| {np.abs(got - fd).max():.2e}"
    closed, mask = padded_closed_form(model, cn, cm)
    assert np.array_equal(AB[:, mask], np.broadcast_to(closed[mask], (B, int(mask.sum()))))
    p.close()


# ---- declarations --------------------------------------------------------------------------------------------------------------------------
def test_rule_declared():
    assert "to_recorded_dims" in K.EXPORTED_SYMBOLS
    lib = K.load_library()
    assert lib.to_recorded_dims.argtypes == [C.c_int32, C.c_int32, K.c_int32_p, K.c_int32_p]
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert "int to_recorded_dims(int32_t nx_max, int32_t nu_max, int32_t* n, int32_t* m);" in hdr
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert "`to_recorded_dims(nx_max, nu_max, &n, &m)`: the smallest of (4, 2), (8, 4) and (16, 8)" in doc
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    assert "function recorded_dims(nx_max::Integer, nu_max::Integer)" in jl
    assert re.search(r"ccall\(\(:to_recorded_dims, libb200\), Cint, \(Int32, Int32, Ref\{Int32\}, Ref\{Int32\}\)", jl)


@pytest.mark.parametrize("lang", ["c", "c++"])
def test_header_compiles(lang):
    src = ("#include \"trajopt_b200.h\"\n"
           "int (*fn)(int32_t, int32_t, int32_t*, int32_t*) = to_recorded_dims;\n"
           "int main(void) { return fn == 0; }\n")
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "l.c" if lang == "c" else "l.cpp")
        open(f, "w").write(src)
        subprocess.check_call(["gcc" if lang == "c" else "g++", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-fsyntax-only", f])
