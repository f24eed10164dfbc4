"""User dynamics programs shared by the CPU and GPU tests of the recorded-program interpreter (csrc/models.cuh dynamics<MODEL_EXPR_42>,
oracle/models.hpp expr_dynamics): programs that between them record every op code, a program at the recording limits, recorded copies
of the built-in models, the NumPy evaluation the oracle is checked against, and malformed program specs the C ABI must reject."""
import numpy as np

import trajopt_b200 as TO

K = TO.capi


# ---- programs that between them record every op code 0..19 -------------------------------------------------------------------------
# every argument stays inside its op's domain for any state and |u| < 3 (rollouts drift away from the drawn states); the tanh
# argument 4 x[0] spans about [-4, 4], so 1 - tanh^2 spans about 1 to 1e-3
def transcendental(x, u):       # n = 4, m = 2
    return [TO.tanh(4.0 * x[0]) * (1.5 - u[1]),
            TO.exp(0.3 * x[2]) / (2.0 + x[3] * x[3]),
            TO.log(1.5 + x[1] * x[1]) + TO.sqrt(2.0 + x[0] * x[0]) - (-x[3]),
            2.0 / (1.0 + u[0] * u[0]) + TO.sin(x[1]) * TO.cos(x[0]) - x[2] * u[1]]


def powers(x, u):               # n = 3, m = 1: exponents 1.5, 0.5, 3, -1, -2.5 (** 2 and ** 1 record no POWC)
    s0 = TO.sin(x[0])
    return [(1.0 + s0 * s0) ** 1.5 + (1.2 + x[1] * x[1]) ** 0.5 - x[2] / 4.0,
            0.1 * (3.0 - u[0]) ** 3 + (1.5 + x[2] * x[2]) ** -1,
            (2.0 + TO.tanh(x[0] * x[1])) ** -2.5 - 0.5]


def constant_rate(x, u):        # n = 2, m = 1: a constant output records OP_CONST
    return [x[1] * u[0], 0.5]


OP_PROGRAMS = {"transcendental": (4, 2, transcendental), "powers": (3, 1, powers), "constant_rate": (2, 1, constant_rate)}


def limit_function(n_instr=TO.capi.EXPR_MAXLEN, n_const=TO.capi.EXPR_MAXCONST):
    """a (4, 2) program that records exactly `n_instr` instructions (6 input loads, the body, the 4 output copies AutodiffDynamics
    appends) and `n_const` constants (the last one is the 1.0 of the output copies)"""
    n_mulc = n_const - 1
    n_fill = n_instr - 6 - n_mulc - 4

    def f(x, u):
        s = list(x)
        for i in range(n_mulc):
            s[i % 4] = s[i % 4] * (1.0 + 0.003 * (i + 1))
        for t in range(n_fill):
            j = t % 4
            if t % 3 == 0:
                s[j] = TO.sin(s[j])
            elif t % 3 == 1:
                s[j] = s[j] * s[(j + 1) % 4]
            else:
                s[j] = s[j] + u[j % 2]
        return s
    return f


def op_model(name, discrete=False):
    if name == "limit":
        return TO.AutodiffDynamics(4, 2, limit_function(), discrete=discrete)
    n, m, f = OP_PROGRAMS[name]
    return TO.AutodiffDynamics(n, m, f, discrete=discrete)


# ---- recorded copies of the built-in models, from the formulas of csrc/models.cuh / oracle/models.hpp -------------------------------
def cartpole_function(mc=1.0, mp=0.2, l=0.5, g=9.81):
    def f(x, u):
        s, c = TO.sin(x[1]), TO.cos(x[1])
        h11, h12, h22 = mc + mp, (mp * l) * c, mp * l * l
        r1 = (-mp * l) * (x[3] * s) * x[3] - u[0]
        r2 = (mp * g * l) * s
        det = h11 * h22 - h12 * h12
        return [x[2], x[3], -(h22 * r1 - h12 * r2) / det, -(h11 * r2 - h12 * r1) / det]
    return f


def acrobot_function(l1=1.0, l2=1.0, m1=1.0, m2=1.0, J1=1.0 / 12.0, J2=1.0 / 12.0, fr=1.0, g=9.81):
    def f(x, u):
        th1, th2, th1d, th2d = x
        c1, s2, c2, c12 = TO.cos(th1), TO.sin(th2), TO.cos(th2), TO.cos(th1 + th2)
        m11 = (m1 * l1 * l1 + J1 + J2) + m2 * ((l1 * l1 + l2 * l2) + (2.0 * l1 * l2) * c2)
        m12 = m2 * ((l2 * l2 + J2) + (l1 * l2) * c2)
        m22 = l2 * l2 * m2 + J2
        tmp = (l1 * l2 * m2) * s2
        b1 = -(2.0 * (th1d * th2d) + th2d * th2d) * tmp
        b2 = tmp * (th1d * th1d)
        f1, f2 = fr * th1d, fr * th2d
        g1 = (((m1 + m2) * l2) * c1 + (m2 * l2) * c12) * g
        g2 = (m2 * l2 * g) * c12
        r1 = -b1 - g1 - f1
        r2 = u[0] - b2 - g2 - f2
        det = m11 * m22 - m12 * m12
        return [th1d, th2d, (m22 * r1 - m12 * r2) / det, (m11 * r2 - m12 * r1) / det]
    return f


def double_integrator_function(dim, mass=1.0):
    return lambda x, u: [x[dim + i] for i in range(dim)] + [u[i] / mass for i in range(dim)]


def recorded_builtin(name):
    """(recorded copy, built-in model) of a built-in model"""
    if name == "cartpole":
        return TO.AutodiffDynamics(4, 1, cartpole_function()), TO.Cartpole()
    if name == "acrobot":
        return TO.AutodiffDynamics(4, 1, acrobot_function()), TO.Acrobot()
    dim = int(name[-1])
    return TO.AutodiffDynamics(2 * dim, dim, double_integrator_function(dim)), TO.DoubleIntegrator(dim)


BUILTINS = ["cartpole", "acrobot", "double_integrator_1", "double_integrator_2"]


def builtin_problem(name, cls, B, recorded, **kw):
    """the problems.py problem of a built-in model, with the built-in model or its recorded copy (Problem(model, ...), same objective,
    constraints, initial state and controls); DiagonalCosts, because problems with recorded dynamics take DiagonalCost / LQRCost"""
    P = TO.problems
    if name == "cartpole":
        ref = P.cartpole(B=B, N=kw.pop("N", 31), cls=cls, u_bound=3.0, goal=True, **kw)
    elif name == "acrobot":
        ref = P.acrobot(B=B, N=kw.pop("N", 51), cls=cls, dense_cost=False, **kw)
    else:
        ref = P.double_integrator(B=B, N=kw.pop("N", 21), dim=int(name[-1]), cls=cls, **kw)
    if not recorded:
        return ref
    rec, _ = recorded_builtin(name)
    tf = float(TO.gettimes(ref)[-1])
    p = cls(rec, ref.obj, ref.x0, tf, xf=ref.xf, constraints=ref.constraints, **kw)
    TO.initial_controls(p, pad(TO.controls(ref), 2))
    return p


# ---- evaluation helpers ---------------------------------------------------------------------------------------------------------------
def pad(a, width):
    """zero-pad the last axis to `width` (the (4, 2) layout of a problem with recorded dynamics)"""
    a = np.asarray(a, dtype=float)
    out = np.zeros(a.shape[:-1] + (width,))
    out[..., :a.shape[-1]] = a
    return out


def numpy_step(model, x, u, h):
    """the model's discrete step evaluated in NumPy from the user's function: the jump map itself, or RK4 with zero-order hold"""
    f = lambda xx: np.array(model.fun(np.asarray(xx, dtype=float), np.asarray(u, dtype=float)), dtype=float)
    if model.discrete:
        return f(x)
    k1 = h * f(x); k2 = h * f(x + 0.5 * k1); k3 = h * f(x + 0.5 * k2); k4 = h * f(x + k3)
    return x + (k1 + 2.0 * k2 + 2.0 * k3 + k4) / 6.0


def numpy_jacobian(model, x, u, h, eps=1e-6):
    """[A B] of numpy_step by central differences"""
    n, m = model.n, model.m
    z = np.concatenate([x, u])
    step = lambda zz: numpy_step(model, zz[:n], zz[n:], h)
    return np.stack([(step(z + e) - step(z - e)) / (2 * eps) for e in eps * np.eye(n + m)], axis=-1)


def one_step_problem(cls, model, B, h=0.1, N=2):
    """a problem of N knots with `model` at every step (Problem(model, ...)) and time step h"""
    obj = TO.LQRObjective(np.ones(model.n), np.ones(model.m), np.ones(model.n), np.zeros(model.n), N)
    return cls(model, obj, np.zeros(model.n), h * (N - 1), batch=B)


def padded_closed_form(model):
    """the rows and columns of the padded (4 x 6) [A B] outside the model's own block: the unused state slots are carried as x+ = x + 0
    by RK4 (identity) and set to zero by a jump map; no state depends on an unused control"""
    AB = np.eye(4, 6) if not model.discrete else np.zeros((4, 6))
    mask = np.ones((4, 6), dtype=bool)
    mask[:model.n_out, :model.n] = False
    mask[:model.n_out, 4:4 + model.m] = False
    return AB, mask


def model_ops(model):
    return set(int(op) for op in np.asarray(model.prog).reshape(-1, 3)[:, 0])


# ---- malformed programs: what to_create / orc_create must reject ----------------------------------------------------------------------
def _base_dyn():
    d = op_model("transcendental")._spec()
    d["prog"] = np.asarray(d["prog"], dtype=np.int32).reshape(-1, 3).copy()
    return d


def malformed_specs(B=2):
    """[(name, Spec, expected code, message fragment)]: valid problem data of 4 knots around one malformed piece"""
    N = 4
    costs = [dict(kind=K.COST_DIAGONAL, Q=np.ones(4), R=np.ones(2), q=np.zeros(4), r=np.zeros(2), c=0.0),
             dict(kind=K.COST_DIAGONAL, Q=np.ones(4), R=np.ones(2), q=np.zeros(4), r=np.zeros(2), c=0.0, terminal=True)]
    base = _base_dyn()
    prog, nconst = base["prog"], len(base["consts"])
    ops = prog[:, 0]
    j_bin = int(np.nonzero((ops >= K.OP_ADD) & (ops <= K.OP_DIV))[0][0])
    j_un = int(np.nonzero(ops == K.OP_TANH)[0][0])
    j_cop = int(np.nonzero(ops == K.OP_ADDC)[0][0])

    def edit(*changes):      # (instruction, column, value) ...
        d = dict(base, prog=base["prog"].copy())
        for j, col, v in changes:
            d["prog"][j, col] = v
        return d

    def spec(dyn=None, dyn_index=(0, 0, 0), nx=(4,) * N, nu=(2,) * N):
        return K.Spec(K.MODEL_EXPR, 4, 2, N, B, np.full(N - 1, 0.1), costs, [0] * (N - 1) + [1], [], dyn=[dyn or base], dyn_index=list(dyn_index),
                      nx=list(nx), nu=list(nu))

    invalid = "recorded-program model: invalid instruction"
    short = dict(base, prog=np.array([[K.OP_X, 0, 0], [K.OP_X, 1, 0], [K.OP_ADD, 0, 1]], dtype=np.int32), consts=np.zeros(0))
    return [
        ("forward register (own result)", spec(edit((j_bin, 2, j_bin))), K.TO_EINVAL, invalid),
        ("forward register (later)", spec(edit((j_un, 1, len(prog) - 1))), K.TO_EINVAL, invalid),
        ("register past the program", spec(edit((j_bin, 1, len(prog) + 7))), K.TO_EINVAL, invalid),
        ("negative register", spec(edit((j_un, 1, -1))), K.TO_EINVAL, invalid),
        ("constant index out of range", spec(edit((j_cop, 2, nconst))), K.TO_EINVAL, invalid),
        ("OP_CONST index out of range", spec(edit((0, 0, K.OP_CONST), (0, 1, nconst))), K.TO_EINVAL, invalid),
        ("op code 20", spec(edit((j_un, 0, 20))), K.TO_EINVAL, invalid),
        ("op code -1", spec(edit((j_un, 0, -1))), K.TO_EINVAL, invalid),
        ("state index out of range", spec(edit((0, 1, 4))), K.TO_EINVAL, invalid),
        ("control index out of range", spec(edit((4, 1, 2))), K.TO_EINVAL, invalid),
        ("n_out > prog_len", spec(short), K.TO_EINVAL, "recorded-program model: bad program size or dimensions"),
        ("n_in != nx", spec(nx=(3, 4, 4, 4)), K.TO_EDIM, "Model 1 has state / control dimensions (4, 2) but knot 1 has (3, 2)."),
        ("m_in != nu", spec(nu=(2, 1, 2, 2)), K.TO_EDIM, "Model 2 has state / control dimensions (4, 2) but knot 2 has (4, 1)."),
        ("dyn_index past the table", spec(dyn_index=(0, 1, 0)), K.TO_EINVAL, "dyn_index out of range"),
        ("negative dyn_index", spec(dyn_index=(0, 0, -1)), K.TO_EINVAL, "dyn_index out of range"),
    ]

