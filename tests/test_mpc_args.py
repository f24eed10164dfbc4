"""Argument checks of the closed-loop MPC calls that happen on the host, before any device call (no GPU needed), and the declarations of
the new entry points and struct in the ctypes binding, the C header, INTEGRATION.md and the Julia shim."""
import ctypes
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _NoDevice:
    """stands in for a Problem: any device call is an error, so a test passes only when the check comes first"""

    def __init__(self, B=4, N=11, model=None, hybrid=False):
        self.model = model if model is not None else TO.Cartpole()
        if hybrid:   # two different recorded models: a hybrid problem
            f = lambda x, u: [x[2], x[3], u[0], u[0]]
            self.model = [TO.AutodiffDynamics(4, 1, f), TO.AutodiffDynamics(4, 1, f)] * ((N - 1) // 2)
        self.hybrid = hybrid
        n, m = (4, 2) if hybrid else self.model.dims()
        self.n, self.m, self.N, self.B = n, m, N, B
        self.ne = n if hybrid else self.model.errstate_dim()
        self.obj = TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n), np.zeros(n), N)

    def _call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _raw_call(self, name, *args):
        raise AssertionError(f"device call {name} reached")

    def _ensure_current(self):
        raise AssertionError("device call reached")


def _ref(p, nref):
    return np.zeros((p.B, nref, p.n)), np.zeros((p.B, nref, p.m))


def test_shapes_raise_dimension_mismatch():
    p = _NoDevice()
    X, U = _ref(p, p.N + 4)
    for kw in [dict(disturbances=np.zeros((4, 5, 3))), dict(disturbances=np.zeros((4, 4, 4))), dict(disturbances=np.zeros((3, 5, 4))),
               dict(plant_params=np.ones((4, 3))), dict(plant_params=np.ones((3, 4))),
               dict(Xref=X[:, :, :3], Uref=U), dict(Xref=X, Uref=U[:2]), dict(Xref=X, Uref=U[:, :-1]), dict(Xref=X[0], Uref=U[0])]:
        with pytest.raises(TO.DimensionMismatch):
            TO.mpc_setup(p, 5, **kw)


def test_reference_too_short():
    """step j = nsteps - 1 tracks rows start - 1 + j .. start - 2 + j + N: the reference must hold start - 1 + (nsteps - 1) + N rows"""
    p = _NoDevice()
    X, U = _ref(p, p.N + 4)                       # 15 rows, N = 11
    TO.api._mpc_inputs(p, 5, None, None, X, U, 1)  # 0 + 4 + 11 = 15: fits
    with pytest.raises(TO.DimensionMismatch, match="shorter"):
        TO.mpc_setup(p, 6, Xref=X, Uref=U)
    with pytest.raises(TO.DimensionMismatch, match="shorter"):
        TO.mpc_setup(p, 5, Xref=X, Uref=U, start=2)
    with pytest.raises(TO.DimensionMismatch, match="shorter"):
        TO.mpc_setup(p, 1, Xref=X, Uref=U, start=0)


@pytest.mark.parametrize("val", [np.nan, np.inf, -np.inf])
def test_non_finite_rows_name_the_instance(val):
    p = _NoDevice()
    X, U = _ref(p, p.N + 4)
    W = np.zeros((4, 5, 4)); W[2, 3, 1] = val
    with pytest.raises(TO.ArgumentError, match="instance 2"):
        TO.mpc_setup(p, 5, disturbances=W)
    X[1, 7, 0] = val
    with pytest.raises(TO.ArgumentError, match="instance 1"):
        TO.mpc_setup(p, 5, Xref=X, Uref=U)
    X[1, 7, 0] = 0.0; U[3, 0, 0] = val
    with pytest.raises(TO.ArgumentError, match="instance 3"):
        TO.mpc_setup(p, 5, Xref=X, Uref=U)
    rows = np.tile(np.asarray(p.model.params, dtype=float), (4, 1)); rows[0, 3] = val
    with pytest.raises(TO.ArgumentError, match="instance 0, parameter 3 is not finite"):
        TO.mpc_setup(p, 5, plant_params=rows)


@pytest.mark.parametrize("model,i", [(TO.Cartpole(), 2), (TO.Quadrotor(), 1), (TO.DoubleIntegrator(1), 0), (TO.Acrobot(), 3)])
def test_plant_rows_set_model_params_would_refuse(model, i):
    """the positive entries of capi.cu positive_param_name: a mass, inertia or length the dynamics divide by"""
    p = _NoDevice(model=model)
    rows = np.tile(np.asarray(model.params, dtype=float), (4, 1)); rows[2, i] = 0.0
    with pytest.raises(TO.ArgumentError, match=f"instance 2, parameter {i} .* must be positive"):
        TO.mpc_setup(p, 3, plant_params=rows)
    # a sequence of models, as set_model_params takes them
    rows = TO.api._mpc_inputs(p, 3, [model] * 4, None, None, None, 1)[1]
    assert rows.shape == (4, len(model.params)) and np.array_equal(rows[1], model.params)


def test_other_refusals_raise_argument_error():
    p = _NoDevice()
    X, U = _ref(p, p.N + 4)
    for bad in (0, -1, 2.5):
        with pytest.raises(TO.ArgumentError, match="nsteps"):
            TO.mpc_setup(p, bad)
    with pytest.raises(TO.ArgumentError, match="together"):
        TO.mpc_setup(p, 2, Xref=X)
    with pytest.raises(TO.ArgumentError, match="together"):
        TO.mpc_setup(p, 2, Uref=U)
    q = _NoDevice()
    q.obj = TO.Objective(TO.AutodiffCost(4, 1, lambda x, u: x[0] * x[0] + u[0] * u[0]), q.N)
    with pytest.raises(TO.ArgumentError, match="QuadraticCostFunctions"):
        TO.mpc_setup(q, 2, Xref=X, Uref=U)


def test_run_and_history_refusals():
    p = _NoDevice()
    with pytest.raises(TO.ArgumentError, match="before mpc_setup"):
        TO.mpc_run(p, 1)
    with pytest.raises(TO.ArgumentError, match="before mpc_setup"):
        TO.mpc_history(p)
    p._mpc = {"nsteps": 5, "done": 3}            # what mpc_setup + mpc_run(3) leave
    for steps, iters in [(0, 1), (1, 0), (-2, 1), (1, -1), (1.5, 1)]:
        with pytest.raises(TO.ArgumentError, match="positive integers"):
            TO.mpc_run(p, steps, iters)
    with pytest.raises(TO.DimensionMismatch, match="3 steps done \\+ 3 exceed the setup's nsteps = 5"):
        TO.mpc_run(p, 3)
    assert p._mpc["done"] == 3


def test_hybrid_problems_refuse():
    p = _NoDevice(hybrid=True)
    with pytest.raises(TO.ArgumentError, match="hybrid"):
        TO.mpc_setup(p, 2)


def test_one_recorded_model_takes_no_reference_or_plant_rows():
    """Problem(AutodiffDynamics(...), ...) steps every knot with one continuous model: a plant like any other, but it has no per-instance
    goals or parameters"""
    f = lambda x, u: [x[2], x[3], u[0], u[0]]
    mdl = TO.AutodiffDynamics(4, 1, f)
    p = _NoDevice(hybrid=True)
    p.model = [mdl] * (p.N - 1)
    nsteps, plant, W, X, U, start = TO.api._mpc_inputs(p, 3, None, np.zeros((4, 3, 4)), None, None, 1)
    assert nsteps == 3 and plant is None and W.shape == (4, 3, 4) and X is None
    Xr, Ur = _ref(p, p.N + 2)
    with pytest.raises(TO.ArgumentError, match="recorded-program"):
        TO.mpc_setup(p, 3, Xref=Xr, Uref=Ur)
    with pytest.raises(TO.ArgumentError, match="recorded-program"):
        TO.mpc_setup(p, 3, plant_params=np.ones((4, 4)))
    jump = TO.AutodiffDynamics(4, 1, f, discrete=True)
    p.model = [jump] * (p.N - 1)
    with pytest.raises(TO.ArgumentError, match="hybrid"):
        TO.mpc_setup(p, 2)


def test_entry_points_declared():
    from trajopt_b200 import capi
    for name in ("to_mpc_setup", "to_mpc_run", "to_mpc_history"):
        assert name in capi.EXPORTED_SYMBOLS
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    assert "int to_mpc_setup(to_handle* h, const to_mpc_spec* spec);" in hdr
    assert "int to_mpc_run(to_handle* h, int32_t steps, int32_t iterations);" in hdr
    assert "int to_mpc_history(to_handle* h, double* Xcl, double* Ucl, double* J);" in hdr
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    for fn in ("function mpc_setup!(p::BatchedProblem", "function mpc_run!(p::BatchedProblem", "function mpc_history(p::BatchedProblem"):
        assert fn in jl
    assert re.search(r"ccall\(\(:to_mpc_run, libb200\), Cint, \(Ptr\{Cvoid\}, Int32, Int32\), p\.h, steps, iterations\)", jl)
    assert callable(TO.mpc_setup) and callable(TO.mpc_run) and callable(TO.mpc_history)
    assert "to_mpc_setup" in open(os.path.join(ROOT, "INTEGRATION.md")).read()


def test_mpc_spec_layout_matches_the_binding_tables():
    """to_mpc_spec's offsets: offsetof / sizeof printed by a C program compiled from include/trajopt_b200.h, against INTEGRATION.md's
    to_mpc_spec table, the ctypes structure and the Julia struct's field order"""
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    body = re.search(r"typedef struct \{((?:(?!typedef struct).)*?)\}\s*to_mpc_spec;", hdr, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            names = decl.split(",")
            fields.append(names[0].split()[-1].lstrip("*"))
            fields += [n.strip().lstrip("*") for n in names[1:]]
    assert fields == ["nsteps", "nparams", "plant_params", "W", "Xref", "Uref", "nref", "start"]
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"trajopt_b200.h\"\nint main() {\n"
    for f in fields:
        src += f'  printf("{f} %zu\\n", offsetof(to_mpc_spec, {f}));\n'
    src += '  printf("sizeof %zu\\n", sizeof(to_mpc_spec));\n  return 0;\n}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "l.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "l.c"), "-o", os.path.join(d, "l")])
        out = subprocess.check_output([os.path.join(d, "l")], text=True)
    c_layout = {l.split()[0]: int(l.split()[1]) for l in out.splitlines()}
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    section = doc[doc.index("### `to_mpc_spec`"):]
    section = section[:section.index("\n## ")]
    table = {m.group(1): int(m.group(2)) for m in re.finditer(r"^\| (\w+) \| (\d+) \|", section, flags=re.M)}
    table["sizeof"] = int(re.search(r"`sizeof\(to_mpc_spec\)` = (\d+)", section).group(1))
    assert table == c_layout
    cls = TO.capi.to_mpc_spec
    assert ctypes.sizeof(cls) == c_layout["sizeof"]
    for f in fields:
        assert getattr(cls, f).offset == c_layout[f], f
    jl = open(os.path.join(ROOT, "trajectoryoptimization.jl_b200", "julia", "B200TrajOpt.jl")).read()
    jbody = re.search(r"struct ToMpcSpec\n(.*?)\nend", jl, flags=re.S).group(1)
    assert re.findall(r"(\w+)::", jbody) == fields
