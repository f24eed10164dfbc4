"""Host-side mirror of the TrajectoryOptimization.jl problem-definition API for the batched H100 hot path.

Same names, argument meaning and error behaviour as the reference's Julia functions (minus the ``!``), so a
user -- or a parity test -- reads like the reference's own code (examples/quickstart.jl).  A ``Problem`` here
is a BATCH of ``B`` independent instances that share model / objective / constraints and differ in ``x0``,
states, controls and multipliers; every numerical call goes through the C ABI (``_capi``) to the sm_90a
kernels.  Nothing in this file computes on the host, except two small pieces of glue that post-process device
results with numpy and say so (``errstate_jacobian``, ``constraint_error_jacobians``).

Array conventions: numpy row-major with the batch first -- ``X[B, N, n]``, ``U[B, N-1, m]`` -- which is the
same memory as Julia's ``Array{Float64,3}(n, N, B)``.  Knot indices given to ``add_constraint`` are 1-based
inclusive ranges exactly like the reference (``add_constraint!(cons, con, 1:N-1)`` -> ``(1, N-1)``).
"""
import ctypes as C
import warnings

import numpy as np

from . import _capi as K
from ._capi import ArgumentError, DimensionMismatch, TrajOptError  # noqa: F401  (re-exported)

# ------------------------------------------------------------------------------------------------------------
# Cones / constraint senses (reference src/cones.jl:17-69)


class ConstraintSense:
    code = None

    def __eq__(self, other):
        return type(self) is type(other)

    def __hash__(self):
        return hash(type(self).__name__)

    def __repr__(self):
        return type(self).__name__ + "()"


class ZeroCone(ConstraintSense):
    code = K.CONE_ZERO


class NegativeOrthant(ConstraintSense):
    code = K.CONE_NEGATIVE_ORTHANT


class SecondOrderCone(ConstraintSense):
    code = K.CONE_SECOND_ORDER


class IdentityCone(ConstraintSense):
    code = K.CONE_IDENTITY


class PositiveOrthant(ConstraintSense):
    code = K.CONE_POSITIVE_ORTHANT


Equality = ZeroCone
Inequality = NegativeOrthant
_CONES = {c.code: c for c in (ZeroCone, NegativeOrthant, SecondOrderCone, IdentityCone, PositiveOrthant)}


def dualcone(cone):   # src/cones.jl:65-69
    return {IdentityCone: ZeroCone, ZeroCone: IdentityCone}.get(type(cone), type(cone))()


_util = None


def _util_handle():
    """A tiny resident problem whose handle serves the stand-alone cone operators."""
    global _util
    if _util is None:
        obj = LQRObjective(np.eye(2), np.eye(1), np.eye(2), np.zeros(2), 2)
        _util = Problem(DoubleIntegrator(1), obj, np.zeros(2), 1.0)
    return _util


def _cone_op(which, cone, x, b=None):
    x = np.ascontiguousarray(np.asarray(x, dtype=np.float64))
    single = x.ndim == 1
    xs = x.reshape(1, -1) if single else x
    count, p = xs.shape
    prob = _util_handle()
    lib = prob._lib
    if which == 0:
        out = np.empty((count, p))
        rc = lib.to_projection(prob._h, cone.code, p, count, K._dp(xs), K._dp(out))
    elif which == 1:
        out = np.empty((count, p, p))
        rc = lib.to_grad_projection(prob._h, cone.code, p, count, K._dp(xs), K._dp(out))
    else:
        bb = np.ascontiguousarray(np.asarray(b, dtype=np.float64)).reshape(count, p)
        out = np.empty((count, p, p))
        rc = lib.to_hess_projection(prob._h, cone.code, p, count, K._dp(xs), K._dp(bb), K._dp(out))
    K.check(lib, prob._h, rc)
    if which > 0:
        out = np.swapaxes(out, -1, -2)   # column-major p x p -> numpy
    return out[0] if single else out


def projection(cone, x):
    """``projection!(cone, px, x)`` (src/cones.jl:96-127) for one vector or a batch ``[count, p]``."""
    return _cone_op(0, cone, x)


def grad_projection(cone, x):
    """``∇projection!(cone, J, x)`` (src/cones.jl:129-188)."""
    return _cone_op(1, cone, x)


def hess_projection(cone, x, b):
    """``∇²projection!(cone, hess, x, b)`` (src/cones.jl:201-276): Hessian of ``x -> Π(x)'b``."""
    return _cone_op(2, cone, x, b)


# ------------------------------------------------------------------------------------------------------------
# Models (RobotZoo / example models; reference docs/src/model.md, examples/Quadrotor.ipynb, examples/quickstart.jl)


class _Model:
    model_id = None
    n = m = None
    params = None

    def dims(self):
        return self.n, self.m

    def errstate_dim(self):   # RD.errstate_dim(model) == state_dim for vector-space models
        return self.n


class DoubleIntegrator(_Model):
    model_id = K.MODEL_DOUBLE_INTEGRATOR

    def __init__(self, dim=1, mass=1.0):
        self.n, self.m, self.params = 2 * dim, dim, [float(mass)]


class Cartpole(_Model):
    model_id = K.MODEL_CARTPOLE
    n, m = 4, 1

    def __init__(self, mc=1.0, mp=0.2, l=0.5, g=9.81):
        self.params = [mc, mp, l, g]


class Quadrotor(_Model):
    model_id = K.MODEL_QUADROTOR
    n, m = 13, 4

    def __init__(self, mass=0.5, J=(0.0023, 0.0023, 0.004), gravity=(0.0, 0.0, -9.81), motor_dist=0.1750, kf=1.0, km=0.0245):
        self.params = [mass, *J, *gravity, motor_dist, kf, km]
        self.mass, self.gravity = mass, gravity

    def errstate_dim(self):
        """``RD.errstate_dim(model)``: the quaternion contributes 3 dimensions (RobotDynamics LieState)."""
        return 12

    def hover_control(self):
        """zeros(model)[2] of RobotZoo.Quadrotor: thrust that cancels gravity (test/internal_api.jl:37)."""
        return np.full(4, -self.gravity[2] * self.mass / 4.0)


class Acrobot(_Model):
    model_id = K.MODEL_ACROBOT
    n, m = 4, 1

    def __init__(self, l=(1.0, 1.0), m=(1.0, 1.0), J=None, friction=1.0, g=9.81):
        J = J or (m[0] * l[0] ** 2 / 12.0, m[1] * l[1] ** 2 / 12.0)
        self.params = [l[0], l[1], m[0], m[1], J[0], J[1], friction, g]


# ------------------------------------------------------------------------------------------------------------
# Cost functions (reference src/cost_functions.jl)


class AutodiffDynamics(_Model):
    """A user-defined dynamics model: the counterpart of ``RD.@autodiff struct M <: RD.ContinuousDynamics end`` + ``RD.state_dim`` /
    ``RD.control_dim`` / ``RD.output_dim`` + ``RD.dynamics(::M, x, u)`` (test/hybrid_dynamics_model.jl:14-39), discretised with RK4 like every
    model of the path (``RD.DiscretizedDynamics{RD.RK4}``).  ``fun(x, u)`` is called once with recording vectors (see ``Expr``) and returns
    the ``output_dim`` entries of ``xdot``.  ``discrete=True``: ``fun`` is a jump map ``x+ = g(x, u)`` applied as is -- its output dimension
    may differ from its state dimension, which is how the state dimension changes along a hybrid trajectory.  Used through
    ``Problem([model_1, ..., model_{N-1}], obj, x0, tf)`` (src/problem.jl:36-73), or on its own as ``Problem(model, obj, x0, tf)``, which is
    ``Problem([model] * (N - 1), obj, x0, tf)``."""
    model_id = K.MODEL_EXPR

    def __init__(self, n, m, fun, output_dim=None, discrete=False):
        self.n, self.m, self.fun, self.discrete = int(n), int(m), fun, bool(discrete)
        self.n_out = self.n if output_dim is None else int(output_dim)
        if self.n_out != self.n and not self.discrete:
            raise ArgumentError("a continuous model integrates its own state: output_dim != state_dim needs discrete=True (a jump map)")
        tape = _Tape("dynamics model")
        x = np.array([tape.emit(K.OP_X, i, 0) for i in range(self.n)], dtype=object)
        u = np.array([tape.emit(K.OP_U, j, 0) for j in range(self.m)], dtype=object)
        out = list(np.atleast_1d(np.asarray(fun(x, u), dtype=object)).ravel())
        if len(out) != self.n_out:
            raise DimensionMismatch(f"the dynamics function returned {len(out)} values, output_dim is {self.n_out}")
        outs = [tape.lift(o) for o in out]
        one = tape.const_index(1.0)
        for o in outs:   # the outputs are the LAST n_out instructions, in order: re-emit each one (x * 1 is exact)
            tape.emit(K.OP_MULC, o.idx, one)
        self.prog, self.consts = np.asarray(tape.prog, dtype=np.int32), np.asarray(tape.consts, dtype=float)

    def output_dim(self):   # RD.output_dim(model)
        return self.n_out

    def copy(self):
        return self

    def _spec(self):
        return dict(n_in=self.n, m_in=self.m, n_out=self.n_out, discrete=self.discrete, prog=self.prog, consts=self.consts)


def model_dims(models):
    """``RD.dims(models::Vector{<:DiscreteDynamics})`` (src/dynamics.jl:15-31): ``(nx, nu)``, the state / control dimension at each of the ``N``
    knot points of ``N - 1`` models; the last state dimension is the last model's output dimension, the last control dimension the last
    model's.  Raises ``DimensionMismatch`` when consecutive models do not fit."""
    models = list(models)
    out = lambda mdl: mdl.output_dim() if hasattr(mdl, "output_dim") else mdl.dims()[0]
    nx = [mdl.dims()[0] for mdl in models] + [out(models[-1])]
    nu = [mdl.dims()[1] for mdl in models] + [models[-1].dims()[1]]
    for k, mdl in enumerate(models, start=1):
        ny = out(mdl)
        if nx[k] != ny:
            raise DimensionMismatch(f"Model mismatch at time step {k}. Model {k} has an output dimension of {ny} but model {k + 1} has a state "
                                    f"dimension of {nx[k]}.")
    return nx, nu


def _isposdef(A):
    A = np.asarray(A, dtype=float)
    if not np.allclose(A, A.T):
        return False
    try:
        np.linalg.cholesky(A)
        return True
    except np.linalg.LinAlgError:
        return False


def _ispossemidef(A):
    A = np.asarray(A, dtype=float)
    return bool(np.all(np.linalg.eigvalsh(0.5 * (A + A.T)) >= -1e-12 * max(1.0, np.abs(A).max())))


def is_diag(cost):   # src/cost_functions.jl:41
    return bool(cost.is_diag)


def is_blockdiag(cost):   # src/cost_functions.jl:48, :382, :455
    return cost.is_blockdiag()


def _isdiag(A):
    A = np.asarray(A, dtype=float)
    return A.ndim == 1 or np.count_nonzero(A - np.diag(np.diagonal(A))) == 0


class CostFunction:
    """``abstract type CostFunction`` (src/cost_functions.jl:8-13): a scalar function of one knot point."""
    is_diag = False


class QuadraticCostFunction(CostFunction):
    """``1/2 x'Qx + 1/2 u'Ru + u'Hx + q'x + r'u + c`` (src/cost_functions.jl:30-58)."""
    is_diag = False

    def __init__(self, Q, R, H=None, q=None, r=None, c=0.0, terminal=False):
        Q, R = np.asarray(Q, dtype=float), np.asarray(R, dtype=float)
        self.Q = np.diag(Q) if Q.ndim == 1 else Q.copy()
        self.R = np.diag(R) if R.ndim == 1 else R.copy()
        n, m = self.Q.shape[0], self.R.shape[0]
        self.H = np.zeros((m, n)) if H is None else np.asarray(H, dtype=float).copy()
        self.q = np.zeros(n) if q is None else np.asarray(q, dtype=float).copy()
        self.r = np.zeros(m) if r is None else np.asarray(r, dtype=float).copy()
        self.c, self.terminal = float(c), bool(terminal)
        if self.q.shape != (n,) or self.r.shape != (m,) or self.H.shape != (m, n):   # asserts at src/cost_functions.jl:434-436
            raise DimensionMismatch("cost function blocks have inconsistent sizes")

    state_dim = property(lambda s: s.Q.shape[0])
    control_dim = property(lambda s: s.R.shape[0])

    def is_blockdiag(self):
        return self.is_diag or np.max(np.abs(self.H), initial=0.0) == 0.0

    def copy(self):   # Base.copy(::DiagonalCost)  src/cost_functions.jl:346-348 (checks = false)
        return type(self)(self.Q, self.R, H=self.H, q=self.q, r=self.r, c=self.c, terminal=self.terminal, checks=False)

    def inv(self):
        """``inv(cost)`` (src/cost_functions.jl:381-383, :471-491): the cost with the inverse Hessian blocks ([Q H'; H R]^-1 when H != 0)."""
        if self.is_diag:
            return DiagonalCost(1.0 / np.diagonal(self.Q), 1.0 / np.diagonal(self.R), q=self.q, r=self.r, c=self.c, terminal=self.terminal, checks=False)
        n = self.state_dim
        if self.is_blockdiag():
            return QuadraticCost(np.linalg.inv(self.Q), np.linalg.inv(self.R), H=self.H, q=self.q, r=self.r, c=self.c, terminal=self.terminal, checks=False)
        G = np.linalg.inv(np.block([[self.Q, self.H.T], [self.H, self.R]]))
        return QuadraticCost(G[:n, :n], G[n:, n:], H=G[n:, :n], q=self.q, r=self.r, c=self.c, terminal=self.terminal, checks=False)

    def __add__(self, other):   # +(c1, c2)  src/cost_functions.jl:259-270
        if isinstance(other, DiagonalQuatCost):
            return other + self   # src/lie_costs.jl:163
        if (self.state_dim, self.control_dim) != (other.state_dim, other.control_dim):
            raise DimensionMismatch("cost functions of different dimensions cannot be added")   # @assert :260-261
        cls = DiagonalCost if (self.is_diag and other.is_diag) else QuadraticCost
        return cls(self.Q + other.Q, self.R + other.R, H=self.H + other.H, q=self.q + other.q, r=self.r + other.r,
                   c=self.c + other.c, terminal=self.terminal and other.terminal, checks=False)

    def _spec(self):
        if self.is_diag:
            return dict(kind=K.COST_DIAGONAL, terminal=self.terminal, Q=np.diag(self.Q).copy(), R=np.diag(self.R).copy(),
                        q=self.q, r=self.r, c=self.c)
        return dict(kind=K.COST_QUADRATIC, terminal=self.terminal, Q=self.Q, R=self.R, H=self.H, q=self.q, r=self.r, c=self.c)


class DiagonalCost(QuadraticCostFunction):   # src/cost_functions.jl:326-347
    is_diag = True

    def __init__(self, Q, R, H=None, q=None, r=None, c=0.0, terminal=False, checks=True):
        super().__init__(Q, R, None, q, r, c, terminal)
        self.Q = np.diag(np.diagonal(self.Q))
        self.R = np.diag(np.diagonal(self.R))
        if checks:   # src/cost_functions.jl:337-343
            if np.any(np.diagonal(self.Q) < 0):
                warnings.warn("Q needs to be positive semi-definite.")
            elif np.any(np.diagonal(self.R) <= 0) and not terminal:
                warnings.warn("R needs to be positive definite.")


class QuadraticCost(QuadraticCostFunction):   # src/cost_functions.jl:417-454
    def __init__(self, Q, R, H=None, q=None, r=None, c=0.0, terminal=False, checks=True):
        super().__init__(Q, R, H, q, r, c, terminal)
        if checks:   # :436-443
            if not terminal and not _isposdef(self.R):
                warnings.warn("R is not positive definite")
            if not _ispossemidef(self.Q):
                warnings.warn("Q is not positive semidefinite")

    def copy(self):
        return QuadraticCost(self.Q, self.R, H=self.H, q=self.q, r=self.r, c=self.c, terminal=self.terminal, checks=False)


class DiagonalQuatCost(DiagonalCost):
    """``DiagonalQuatCost(Q, R, q, r, c, w, q_ref, q_ind)`` (src/lie_costs.jl:33-56):
    ``1/2 x'Qx + 1/2 u'Ru + q'x + r'u + c + w min(1 + q_ref'p, 1 - q_ref'p)`` with ``p = x[q_ind]`` (1-based indices, default 4:7)."""

    def __init__(self, Q, R, q=None, r=None, c=0.0, w=1.0, q_ref=(1.0, 0.0, 0.0, 0.0), q_ind=(4, 5, 6, 7), terminal=False):
        super().__init__(Q, R, None, q, r, c, terminal)
        self.w = float(w)
        self.q_ref = np.asarray(q_ref, dtype=float).copy()
        self.q_ind = np.asarray(q_ind, dtype=int).copy()
        if self.q_ref.shape != (4,) or self.q_ind.shape != (4,):
            raise DimensionMismatch("quat_ind argument must be of length 4")   # @assert src/lie_costs.jl:132
        if self.q_ind.min() < 1 or self.q_ind.max() > self.state_dim:
            raise DimensionMismatch("DiagonalQuatCost: q_ind outside the state")

    def copy(self):   # Base.copy  src/lie_costs.jl:165-167
        return DiagonalQuatCost(self.Q, self.R, q=self.q, r=self.r, c=self.c, w=self.w, q_ref=self.q_ref, q_ind=self.q_ind, terminal=self.terminal)

    def __add__(self, other):   # +(::DiagonalQuatCost, ::QuadraticCostFunction)  src/lie_costs.jl:152-163
        if not other.is_diag and np.max(np.abs(other.H), initial=0.0) != 0.0:
            raise ArgumentError("DiagonalQuatCost + cost with a non-zero H")   # @assert norm(cost2.H) ~ 0
        return DiagonalQuatCost(self.Q + other.Q, self.R + other.R, q=self.q + other.q, r=self.r + other.r, c=self.c + other.c,
                                w=self.w, q_ref=self.q_ref, q_ind=self.q_ind)

    __radd__ = __add__

    def _spec(self):
        d = super()._spec()
        d.update(kind=K.COST_DIAGONAL_QUAT, w=self.w, q_ref=self.q_ref, q_ind=self.q_ind)
        return d


def QuatLQRCost(Q, R, xf, uf=None, w=1.0, quat_ind=(4, 5, 6, 7), **kw):
    """``QuatLQRCost(Q, R, xf, uf; w, quat_ind)`` (src/lie_costs.jl:129-139)."""
    Q, R = np.asarray(Q, dtype=float), np.asarray(R, dtype=float)
    Qm = np.diag(Q) if Q.ndim == 1 else Q
    Rm = np.diag(R) if R.ndim == 1 else R
    xf = np.asarray(xf, dtype=float)
    uf = np.zeros(Rm.shape[0]) if uf is None else np.asarray(uf, dtype=float)
    quat_ind = np.asarray(quat_ind, dtype=int)
    if quat_ind.size != 4:
        raise DimensionMismatch("quat_ind argument must be of length 4")
    return DiagonalQuatCost(Qm, Rm, q=-Qm @ xf, r=-Rm @ uf, c=0.5 * xf @ Qm @ xf + 0.5 * uf @ Rm @ uf, w=w, q_ref=xf[quat_ind - 1],
                            q_ind=quat_ind, **kw)


# ---- user-defined costs: RD.@autodiff struct ... <: CostFunction (docs/src/costfunction_interface.md:30-50, test/nlcosts.jl:4-19) ----


class Expr:
    """One value of a recorded straight-line program.  Calling the user's cost function on vectors of ``Expr`` records the
    arithmetic it performs (what ForwardDiff's dual numbers see in the reference); the device evaluates the recording with
    second-order forward-mode duals.  Supports + - * / **const, unary -, and sin cos exp log sqrt tanh (also through numpy ufuncs)."""
    __array_priority__ = 1000

    def __init__(self, tape, idx):
        self.tape, self.idx = tape, idx

    def _bin(self, other, op, swap=False):
        if not isinstance(other, Expr):   # a plain number: one instruction with a constant-table operand
            c = float(other)
            if op == K.OP_ADD: return self.tape.emit(K.OP_ADDC, self.idx, self.tape.const_index(c))
            if op == K.OP_MUL: return self.tape.emit(K.OP_MULC, self.idx, self.tape.const_index(c))
            if op == K.OP_SUB: return self.tape.emit(K.OP_RSUBC if swap else K.OP_ADDC, self.idx, self.tape.const_index(c if swap else -c))
            if op == K.OP_DIV: return self.tape.emit(K.OP_RDIVC if swap else K.OP_DIVC, self.idx, self.tape.const_index(c))
        o = self.tape.lift(other)
        a, b = (o, self) if swap else (self, o)
        return self.tape.emit(op, a.idx, b.idx)

    __add__ = lambda s, o: s._bin(o, K.OP_ADD)
    __radd__ = lambda s, o: s._bin(o, K.OP_ADD, True)
    __sub__ = lambda s, o: s._bin(o, K.OP_SUB)
    __rsub__ = lambda s, o: s._bin(o, K.OP_SUB, True)
    __mul__ = lambda s, o: s._bin(o, K.OP_MUL)
    __rmul__ = lambda s, o: s._bin(o, K.OP_MUL, True)
    __truediv__ = lambda s, o: s._bin(o, K.OP_DIV)
    __rtruediv__ = lambda s, o: s._bin(o, K.OP_DIV, True)
    __neg__ = lambda s: s.tape.emit(K.OP_NEG, s.idx, 0)
    __pos__ = lambda s: s

    def __pow__(self, e):
        if isinstance(e, Expr):
            raise ArgumentError("Expr ** Expr is not recorded: use exp(e * log(x))")
        e = float(e)
        if e == 2.0:
            return self * self
        if e == 1.0:
            return self
        return self.tape.emit(K.OP_POWC, self.idx, self.tape.const_index(e))

    def _un(self, op):
        return self.tape.emit(op, self.idx, 0)

    sin = lambda s: s._un(K.OP_SIN)
    cos = lambda s: s._un(K.OP_COS)
    exp = lambda s: s._un(K.OP_EXP)
    log = lambda s: s._un(K.OP_LOG)
    sqrt = lambda s: s._un(K.OP_SQRT)
    tanh = lambda s: s._un(K.OP_TANH)

    def __bool__(self):
        raise ArgumentError(f"a recorded {self.tape.what} cannot branch on a state / control value")


class _Tape:
    def __init__(self, what):
        self.what = what     # what is being recorded ("cost", "dynamics model", "constraint"), for the error messages
        self.prog, self.consts = [], []

    def emit(self, op, a, b):
        if len(self.prog) >= K.EXPR_MAXLEN:
            raise ArgumentError(f"recorded {self.what} exceeds {K.EXPR_MAXLEN} instructions")
        self.prog.append((int(op), int(a), int(b)))
        return Expr(self, len(self.prog) - 1)

    def const_index(self, v):
        v = float(v)
        for i, c in enumerate(self.consts):
            if c == v and np.signbit(c) == np.signbit(v):
                return i
        if len(self.consts) >= K.EXPR_MAXCONST:
            raise ArgumentError(f"recorded {self.what} exceeds {K.EXPR_MAXCONST} constants")
        self.consts.append(v)
        return len(self.consts) - 1

    def lift(self, v):
        if isinstance(v, Expr):
            if v.tape is not self:
                raise ArgumentError("mixing values of two recordings")
            return v
        return self.emit(K.OP_CONST, self.const_index(v), 0)


def sin(x): return x.sin() if isinstance(x, Expr) else np.sin(x)
def cos(x): return x.cos() if isinstance(x, Expr) else np.cos(x)
def exp(x): return x.exp() if isinstance(x, Expr) else np.exp(x)
def log(x): return x.log() if isinstance(x, Expr) else np.log(x)
def sqrt(x): return x.sqrt() if isinstance(x, Expr) else np.sqrt(x)
def tanh(x): return x.tanh() if isinstance(x, Expr) else np.tanh(x)


class AutodiffCost(CostFunction):
    """A user-defined cost ``fun(x, u) -> scalar``: the counterpart of ``RD.@autodiff struct MyCost <: CostFunction`` +
    ``RD.evaluate(cost, x, u)`` (docs/src/costfunction_interface.md:30-50; test/nlcosts.jl:4-19).  ``fun`` is called once with
    recording vectors (``x[i]``, ``u[j]`` 0-based, numpy object arrays: ``x @ Q @ x``, ``np.cos(x[1] / 2)``, ``TO.cos`` all work);
    gradient and Hessian come from forward-mode automatic differentiation of the recording on the device, like ``ForwardAD()``.
    At the terminal knot the cost is evaluated with ``u = 0`` and only its state derivatives are used."""

    def __init__(self, n, m, fun, terminal=False):
        self.n, self.m, self.fun, self.terminal = int(n), int(m), fun, bool(terminal)
        tape = _Tape("cost")
        x = np.array([tape.emit(K.OP_X, i, 0) for i in range(self.n)], dtype=object)
        u = np.array([tape.emit(K.OP_U, j, 0) for j in range(self.m)], dtype=object)
        out = fun(x, u)
        out = tape.lift(out if not isinstance(out, np.ndarray) else out.item())
        if out.idx != len(tape.prog) - 1:          # the result must be the last instruction: re-emit it
            out = tape.emit(K.OP_ADD, out.idx, tape.lift(0.0).idx)
        self.prog, self.consts = np.asarray(tape.prog, dtype=np.int32), np.asarray(tape.consts, dtype=float)

    state_dim = property(lambda s: s.n)
    control_dim = property(lambda s: s.m)

    def copy(self):
        return AutodiffCost(self.n, self.m, self.fun, self.terminal)

    def _spec(self):
        return dict(kind=K.COST_EXPR, terminal=self.terminal, prog=self.prog, consts=self.consts)


def ErrorQuadratic(model, Q, R, x_ref, u_ref=None, r=None, c=0.0, q_ind=(4, 5, 6, 7), terminal=False):
    """``ErrorQuadratic(model, Q, R, x_ref, u_ref; r, c, q_ind)`` (src/lie_costs.jl:170-240): ``1/2 dx'Q dx + c + 1/2 u'Ru + r'u`` with
    ``dx = RD.state_diff(model, x, x_ref, CayleyMap())`` the 12-dimensional error state of a rigid body (``Q`` of the full state size
    loses its 4th entry, :214-217; ``r -= R u_ref``, ``c += 1/2 u_ref'R u_ref``, :218-219).  The reference differentiates it with
    ForwardAD (:196); here it is a recorded program (``AutodiffCost``).  The reference's own advice (:185-186): prefer ``DiagonalQuatCost``."""
    n, m = model.dims()
    if model.errstate_dim() == n:
        raise ArgumentError("ErrorQuadratic needs a rigid-body (Lie-group) model")
    Qd = np.asarray(Q, dtype=float)
    Qd = np.diag(Qd).copy() if Qd.ndim == 2 else Qd.copy()
    Rd = np.asarray(R, dtype=float)
    Rd = np.diag(Rd).copy() if Rd.ndim == 2 else Rd.copy()
    x_ref = np.asarray(x_ref, dtype=float)
    q_ind = np.asarray(q_ind, dtype=int) - 1
    if Qd.size == x_ref.size:
        Qd = np.delete(Qd, q_ind[0])
    if Qd.size != n - 1 or Rd.size != m:
        raise DimensionMismatch("ErrorQuadratic: Q must have 12 (or 13) and R m diagonal entries")
    u_ref = np.zeros(m) if u_ref is None else np.asarray(u_ref, dtype=float)
    rv = (np.zeros(m) if r is None else np.asarray(r, dtype=float)) - Rd * u_ref
    cc = float(c) + 0.5 * float(u_ref @ (Rd * u_ref))
    qr = x_ref[q_ind]
    vec_idx = [i for i in range(n) if i not in set(q_ind.tolist())]

    def fun(x, u):
        # state_diff: q_ref^-1 (x) q, inverse Cayley map = vector part / scalar part; vector states subtract
        p = [x[i] for i in q_ind]
        dw = qr[0] * p[0] + qr[1] * p[1] + qr[2] * p[2] + qr[3] * p[3]
        dv = [qr[0] * p[1] - qr[1] * p[0] - (qr[2] * p[3] - qr[3] * p[2]),
              qr[0] * p[2] - qr[2] * p[0] - (qr[3] * p[1] - qr[1] * p[3]),
              qr[0] * p[3] - qr[3] * p[0] - (qr[1] * p[2] - qr[2] * p[1])]
        dx = [x[i] - x_ref[i] for i in vec_idx[:q_ind[0]]] + [d / dw for d in dv] + [x[i] - x_ref[i] for i in vec_idx[q_ind[0]:]]
        J = None
        for w, d in zip(Qd, dx):
            if w != 0.0:
                t = w * (d * d)
                J = t if J is None else J + t
        for w, rr, uu in zip(Rd, rv, u):
            if w != 0.0:
                t = w * (uu * uu)
                J = t if J is None else J + t
        J = 0.5 * J if J is not None else 0.0
        for rr, uu in zip(rv, u):
            if rr != 0.0:
                J = J + rr * uu
        return J + cc if cc != 0.0 else J
    return AutodiffCost(n, m, fun, terminal=terminal)


def make_quadratic_cost(Q, R, H=None, q=None, r=None, c=0.0, **kw):
    """``QuadraticCostFunction(Q,R,H,q,r,c)`` (src/cost_functions.jl:60-68): Diagonal when it can be."""
    Hn = 0.0 if H is None else float(np.max(np.abs(H), initial=0.0))
    cls = DiagonalCost if (_isdiag(Q) and _isdiag(R) and Hn == 0.0) else QuadraticCost
    return cls(Q, R, H=H, q=q, r=r, c=c, **kw)


def set_LQR_goal(cost, xf, uf=None):   # set_LQR_goal!  src/cost_functions.jl:245-254 (c is left as is)
    cost.q = -cost.Q @ np.asarray(xf, dtype=float)
    if uf is not None:
        cost.r = -cost.R @ np.asarray(uf, dtype=float)
    cost._version = getattr(cost, "_version", 0) + 1      # a live Problem holding this cost re-uploads its tables before the next device call


def LQRCost(Q, R, xf, uf=None, **kw):   # src/cost_functions.jl:532-547
    Q, R = np.asarray(Q, dtype=float), np.asarray(R, dtype=float)
    Qm = np.diag(Q) if Q.ndim == 1 else Q
    Rm = np.diag(R) if R.ndim == 1 else R
    xf = np.asarray(xf, dtype=float)
    uf = np.zeros(Rm.shape[0]) if uf is None else np.asarray(uf, dtype=float)
    return make_quadratic_cost(Qm, Rm, None, -Qm @ xf, -Rm @ uf, 0.5 * xf @ Qm @ xf + 0.5 * uf @ Rm @ uf, **kw)


class Objective:
    """``Objective`` (src/objective.jl:27-45): one cost function per knot point."""

    def __init__(self, cost, *args):
        if isinstance(cost, CostFunction) and len(args) == 1:                   # Objective(cost, N)       :69-71
            self.cost = [cost for _ in range(int(args[0]))]
        elif isinstance(cost, CostFunction) and len(args) == 2:                 # Objective(cost, term, N) :73-76
            N = int(args[1])
            self.cost = [cost if k < N - 1 else args[0] for k in range(N)]
        elif len(args) == 1:                                                     # Objective(costs, term)   :78-81
            self.cost = list(cost) + [args[0]]
        else:
            self.cost = list(cost)
        self.J = np.zeros(len(self.cost))     # (costs of different dimensions are allowed: hybrid problems, RD.dims(obj) src/objective.jl:49)

    def __len__(self):
        return len(self.cost)

    def __getitem__(self, k):
        return self.cost[k]

    def __iter__(self):
        return iter(self.cost)

    def dims(self):
        return self.cost[0].state_dim, self.cost[0].control_dim

    def dims_all(self):   # RD.dims(obj)  src/objective.jl:49: per-knot dimensions
        return [c.state_dim for c in self.cost], [c.control_dim for c in self.cost]

    def copy(self):   # Base.copy(obj)  src/objective.jl:112: copies of the cost functions (knots that share a cost object keep sharing the copy)
        memo = {}
        return Objective([memo.setdefault(id(c), c.copy()) for c in self.cost])

    def _tables(self):
        """distinct cost objects + per-knot index (what the device cost table holds)."""
        uniq, index, seen = [], [], {}
        for c in self.cost:
            if id(c) not in seen:
                seen[id(c)] = len(uniq)
                uniq.append(c)
            index.append(seen[id(c)])
        return uniq, index


def LQRObjective(Q, R, Qf, xf, N, uf=None):
    """``LQRObjective(Q, R, Qf, xf, N; uf)`` (src/objective.jl:137-183): the terminal cost keeps R and r."""
    Q, R, Qf = (np.asarray(a, dtype=float) for a in (Q, R, Qf))
    Qm, Rm, Qfm = (np.diag(a) if a.ndim == 1 else a for a in (Q, R, Qf))
    xf = np.asarray(xf, dtype=float)
    if Qm.shape[0] != xf.size or Qfm.shape[0] != xf.size:
        raise DimensionMismatch("Q / Qf size does not match xf")   # @assert src/objective.jl:141-143
    uf = np.zeros(Rm.shape[0]) if uf is None else np.asarray(uf, dtype=float)
    if Rm.shape[0] != uf.size:
        raise DimensionMismatch("R size does not match uf")
    q, r = -Qm @ xf, -Rm @ uf
    c = 0.5 * xf @ Qm @ xf + 0.5 * uf @ Rm @ uf
    qf, cf = -Qfm @ xf, 0.5 * xf @ Qfm @ xf
    diag = _isdiag(Qm) and _isdiag(Rm) and _isdiag(Qfm)
    cls = DiagonalCost if diag else QuadraticCost
    stage = cls(Qm, Rm, q=q, r=r, c=c)
    term = cls(Qfm, Rm, q=qf, r=r, c=cf, terminal=True)
    return Objective(stage, term, N)


def TrackingObjective(Q, R, X, U, Qf=None):
    """``TrackingObjective(Q, R, Z; Qf)`` (src/objective.jl:190-196); ``X[N,n]``, ``U[N-1,m]`` reference trajectory."""
    X, U = np.asarray(X, dtype=float), np.asarray(U, dtype=float)
    N = X.shape[0]
    costs = [LQRCost(Q, R, X[k], U[k]) for k in range(N - 1)]
    costs.append(LQRCost(Q if Qf is None else Qf, R, X[N - 1], terminal=True))
    return Objective(costs)


# ------------------------------------------------------------------------------------------------------------
# Constraints (reference src/constraints.jl, src/abstract_constraint.jl, src/constraint_list.jl)


class AbstractConstraint:
    sense_ = Inequality()

    def _spec(self, first, last):
        raise NotImplementedError


def sense(con):   # src/abstract_constraint.jl:97
    return con.sense_


def output_dim(con):
    return con.p


def is_bound(con):   # src/abstract_constraint.jl:139
    if isinstance(con, IndexedConstraint):   # src/constraints.jl:930
        return is_bound(con.con)
    return isinstance(con, (GoalConstraint, BoundConstraint))


def upper_bound(con):   # src/abstract_constraint.jl:104-109
    if isinstance(con, IndexedConstraint): return upper_bound(con.con)   # src/constraints.jl:931
    if isinstance(con, StateBound): return con.x_max.copy()        # src/constraints.jl:607
    if isinstance(con, ControlBound): return con.u_max.copy()      # :630
    if isinstance(con, BoundConstraint):
        return con.z_max.copy()      # src/constraints.jl:733
    return np.full(con.p, {ZeroCone: 0.0, NegativeOrthant: 0.0}.get(type(con.sense_), np.inf))


def lower_bound(con):   # src/abstract_constraint.jl:116-121
    if isinstance(con, IndexedConstraint): return lower_bound(con.con)   # src/constraints.jl:932
    if isinstance(con, StateBound): return con.x_min.copy()        # src/constraints.jl:606
    if isinstance(con, ControlBound): return con.u_min.copy()      # :629
    if isinstance(con, BoundConstraint):
        return con.z_min.copy()      # src/constraints.jl:732
    return np.full(con.p, {ZeroCone: 0.0}.get(type(con.sense_), -np.inf))


class GoalConstraint(AbstractConstraint):   # src/constraints.jl:22-87
    sense_ = Equality()

    def __init__(self, xf, inds=None):
        xf = np.asarray(xf, dtype=float)
        self.n = xf.size
        self.inds = np.arange(1, self.n + 1) if inds is None else np.asarray(inds, dtype=int)
        self.xf = xf[self.inds - 1].copy()
        self.p = self.inds.size

    def _spec(self, first, last):
        return dict(kind=K.CON_GOAL, first=first, last=last, sense=K.CONE_ZERO, inds=self.inds, a=self.xf)


def _check_bounds(k, hi, lo):   # checkBounds  src/constraints.jl:708-719
    hi = np.full(k, float(hi)) if np.ndim(hi) == 0 else np.asarray(hi, dtype=float)
    lo = np.full(k, float(lo)) if np.ndim(lo) == 0 else np.asarray(lo, dtype=float)
    if not np.all(hi >= lo):
        raise ArgumentError("Upper bounds must be greater than or equal to lower bounds")
    return hi, lo


class BoundConstraint(AbstractConstraint):   # src/constraints.jl:644-783
    sense_ = Inequality()

    def __init__(self, n, m, x_min=-np.inf, x_max=np.inf, u_min=-np.inf, u_max=np.inf):
        self.n, self.m = n, m
        x_max, x_min = _check_bounds(n, x_max, x_min)
        u_max, u_min = _check_bounds(m, u_max, u_min)
        self.z_max, self.z_min = np.concatenate([x_max, u_max]), np.concatenate([x_min, u_min])
        self.p = int(np.isfinite(self.z_max).sum() + np.isfinite(self.z_min).sum())

    def _spec(self, first, last):
        return dict(kind=K.CON_BOUND, first=first, last=last, sense=K.CONE_NEGATIVE_ORTHANT, a=self.z_max, b=self.z_min)


class LinearConstraint(AbstractConstraint):   # src/constraints.jl:103-150
    def __init__(self, n, m, A, b, sense, inds="state"):
        self.n, self.m = n, m
        self.A, self.b = np.atleast_2d(np.asarray(A, dtype=float)), np.asarray(b, dtype=float)
        self.on_control = inds in ("control", 1)
        self.p, self.sense_ = self.A.shape[0], sense
        if self.A.shape[1] != (m if self.on_control else n) or self.b.size != self.p:
            raise DimensionMismatch("LinearConstraint: A / b size mismatch")   # @assert src/constraints.jl:113-116

    def _spec(self, first, last):
        return dict(kind=K.CON_LINEAR, first=first, last=last, sense=self.sense_.code, p=self.p, flag=int(self.on_control), a=self.A, b=self.b)


class CircleConstraint(AbstractConstraint):   # src/constraints.jl:168-233
    def __init__(self, n, xc, yc, radius, xi=1, yi=2):
        self.n = n
        self.x, self.y, self.radius = (np.atleast_1d(np.asarray(a, dtype=float)) for a in (xc, yc, radius))
        self.xi, self.yi, self.p = xi, yi, self.x.size

    def _spec(self, first, last):
        return dict(kind=K.CON_CIRCLE, first=first, last=last, sense=K.CONE_NEGATIVE_ORTHANT, p=self.p, a=self.x, b=self.y,
                    rad=self.radius, inds=[self.xi, self.yi])


class SphereConstraint(AbstractConstraint):   # src/constraints.jl:249-326
    def __init__(self, n, xc, yc, zc, radius, xi=1, yi=2, zi=3):
        self.n = n
        self.x, self.y, self.z, self.radius = (np.atleast_1d(np.asarray(a, dtype=float)) for a in (xc, yc, zc, radius))
        self.xi, self.yi, self.zi, self.p = xi, yi, zi, self.x.size

    def _spec(self, first, last):
        return dict(kind=K.CON_SPHERE, first=first, last=last, sense=K.CONE_NEGATIVE_ORTHANT, p=self.p, a=self.x, b=self.y, c=self.z,
                    rad=self.radius, inds=[self.xi, self.yi, self.zi])


class NormConstraint(AbstractConstraint):   # src/constraints.jl:438-521
    def __init__(self, n, m, val, sense, inds="all"):
        self.n, self.m, self.val, self.sense_ = n, m, float(val), sense
        if isinstance(inds, str):   # src/constraints.jl:446-454
            inds = {"state": range(1, n + 1), "control": range(n + 1, n + m + 1), "all": range(1, n + m + 1)}[inds]
        self.inds = np.asarray(list(inds), dtype=int)
        if self.val < 0:
            raise ArgumentError("NormConstraint value must be non-negative")   # @assert val >= 0 src/constraints.jl:443
        self.p = self.inds.size + 1 if isinstance(sense, SecondOrderCone) else 1

    def _spec(self, first, last):
        return dict(kind=K.CON_NORM, first=first, last=last, sense=self.sense_.code, val=self.val, inds=self.inds)


class CollisionConstraint(AbstractConstraint):   # src/constraints.jl:328-389
    """``CollisionConstraint(n, x1, x2, r)``: ``r^2 - |x[x1] - x[x2]|^2 <= 0`` (1-based state indices)."""

    def __init__(self, n, x1, x2, radius):
        self.n = n
        self.x1, self.x2 = np.asarray(list(x1), dtype=int), np.asarray(list(x2), dtype=int)
        if self.x1.size != self.x2.size:
            raise DimensionMismatch(f"Position dimensions must be of equal length, got {self.x1.size} and {self.x2.size}")   # @assert :349
        self.radius, self.p = float(radius), 1

    def _spec(self, first, last):
        return dict(kind=K.CON_COLLISION, first=first, last=last, sense=K.CONE_NEGATIVE_ORTHANT, val=self.radius,
                    inds=np.concatenate([self.x1, self.x2]))


class QuatVecEq(AbstractConstraint):   # src/constraints.jl:938-965
    """``QuatVecEq(n, m, qf, qind=4:7)``: the vector part of the normalised quaternion ``x[qind]`` equals that of ``qf`` (sign-matched)."""
    sense_ = Equality()

    def __init__(self, n, m, qf, qind=(4, 5, 6, 7)):
        self.n, self.m = n, m
        self.qf = np.asarray(qf, dtype=float).copy()
        self.qind = np.asarray(qind, dtype=int).copy()
        if self.qf.shape != (4,) or self.qind.shape != (4,):
            raise DimensionMismatch("QuatVecEq: qf and qind must have 4 entries")
        self.p = 3

    def _spec(self, first, last):
        return dict(kind=K.CON_QUATVEC, first=first, last=last, sense=K.CONE_ZERO, a=self.qf, inds=self.qind)


class AutodiffConstraint(AbstractConstraint):
    """A user-defined constraint ``fun(x, u) -> p values``: the counterpart of ``RD.@autodiff struct MyCon <: StageConstraint`` with
    ``RD.evaluate(con, x, u)`` (docs/src/constraint_interface.md:52-72).  ``inputs`` = ``"stage"`` (``fun(x, u)``), ``"state"``
    (``fun(x)``, a ``StateConstraint``) or ``"control"`` (``fun(u)``, a ``ControlConstraint``).  ``fun`` is recorded once (see ``Expr``);
    values and the forward-mode Jacobian are evaluated on the device."""

    def __init__(self, n, m, fun, sense, inputs="stage"):
        self.n, self.m, self.fun, self.sense_, self.inputs = int(n), int(m), fun, sense, inputs
        tape = _Tape("constraint")
        x = np.array([tape.emit(K.OP_X, i, 0) for i in range(self.n)], dtype=object)
        u = np.array([tape.emit(K.OP_U, j, 0) for j in range(self.m)], dtype=object)
        out = fun(x, u) if inputs == "stage" else (fun(x) if inputs == "state" else fun(u))
        outs = [tape.lift(o) for o in np.atleast_1d(np.asarray(out, dtype=object)).ravel()]
        outs = [tape.emit(K.OP_ADDC, o.idx, tape.const_index(0.0)) for o in outs]      # the outputs are the last p instructions, in order
        self.p = len(outs)
        if self.p < 1 or self.p > 16:
            raise ArgumentError("the solver kernels take 1..16 rows per general constraint")
        self.prog, self.consts = np.asarray(tape.prog, dtype=np.int32), np.asarray(tape.consts, dtype=float)

    def _spec(self, first, last):
        return dict(kind=K.CON_EXPR, first=first, last=last, sense=self.sense_.code, p=self.p, inds=self.prog.ravel(), a=self.consts,
                    flag=len(self.consts))


def _index_vec(idx, default_len):
    """1-based index vector from a Julia-style range ``(first, last)``, a list, or None (= 1:default_len)."""
    if idx is None:
        return np.arange(1, default_len + 1)
    if isinstance(idx, tuple) and len(idx) == 2:
        return np.arange(int(idx[0]), int(idx[1]) + 1)
    return np.asarray(list(idx), dtype=int)


class IndexedConstraint(AbstractConstraint):
    """``IndexedConstraint(n, m, con, ix, iu)`` (src/constraints.jl:785-936): ``con``, defined for a model with ``(n0, m0)``, applied to
    the slices ``x[ix]``, ``u[iu]`` of a larger model ``(n, m)`` (1-based, increasing indices; a ``(first, last)`` tuple is a Julia range).
    Host-side only: the indices are remapped and the same device constraint kinds are used."""

    def __init__(self, n, m, con, ix=None, iu=None):
        if isinstance(con, IndexedConstraint):
            raise ArgumentError("nested IndexedConstraint")
        self.n, self.m, self.con = int(n), int(m), con
        n0 = getattr(con, "n", None)
        m0 = getattr(con, "m", None)
        if isinstance(con, StateBound): m0 = 0 if m0 is None else m0
        if isinstance(con, ControlBound): n0 = 0 if n0 is None else n0
        self.ix = _index_vec(ix, n0 if n0 is not None else n)       # IndexedConstraint(n, m, con): start of the vectors (:882-897)
        self.iu = _index_vec(iu, m0 if m0 is not None else m)
        self.n0, self.m0 = (self.ix.size if n0 is None else n0), (self.iu.size if m0 is None else m0)
        if (n0 not in (None, 0) and self.ix.size != n0) or (m0 not in (None, 0) and self.iu.size != m0):
            raise DimensionMismatch("IndexedConstraint: ix / iu do not match the dimensions of the wrapped constraint")
        if self.ix.size and (self.ix.min() < 1 or self.ix.max() > n or np.any(np.diff(self.ix) <= 0)):
            raise ArgumentError("IndexedConstraint: ix must be increasing indices into 1:n")
        if self.iu.size and (self.iu.min() < 1 or self.iu.max() > m or np.any(np.diff(self.iu) <= 0)):
            raise ArgumentError("IndexedConstraint: iu must be increasing indices into 1:m")
        self.p, self.sense_ = con.p, con.sense_

    def _zmap(self, j):
        """1-based index into the old z = [x0; u0] -> 1-based index into the new z"""
        return int(self.ix[j - 1]) if j <= self.n0 else self.n + int(self.iu[j - self.n0 - 1])

    def _spec(self, first, last):
        con = self.con
        if isinstance(con, (StateBound, ControlBound)):
            con._bind(self.m0 if isinstance(con, StateBound) else self.n0)
        d = dict(con._spec(first, last))
        k = d["kind"]
        if k == K.CON_BOUND:      # change_dimension(::BoundConstraint) :772-783 (which fills x_min with +Inf: the intended -Inf is used here)
            zmax, zmin = np.full(self.n + self.m, np.inf), np.full(self.n + self.m, -np.inf)
            n0 = self.n0
            for j in range(con.z_max.size):
                jj = (int(self.ix[j]) - 1) if j < n0 else self.n + int(self.iu[j - n0]) - 1
                zmax[jj], zmin[jj] = con.z_max[j], con.z_min[j]
            d.update(a=zmax, b=zmin)
        elif k == K.CON_LINEAR:   # :146-150
            src = self.iu if d["flag"] else self.ix
            A = np.zeros((con.p, self.m if d["flag"] else self.n))
            A[:, src - 1] = con.A
            d.update(a=A)
        elif k in (K.CON_GOAL, K.CON_CIRCLE, K.CON_SPHERE, K.CON_COLLISION, K.CON_QUATVEC):   # state indices (:75, :231, :324, :391)
            d.update(inds=[int(self.ix[j - 1]) for j in np.asarray(d["inds"], dtype=int)])
        elif k == K.CON_NORM:     # indices into z (:519)
            d.update(inds=[self._zmap(int(j)) for j in np.asarray(d["inds"], dtype=int)])
        elif k == K.CON_EXPR:     # recorded program: remap the loads
            prog = np.asarray(d["inds"], dtype=np.int32).reshape(-1, 3).copy()
            for row in prog:
                if row[0] == K.OP_X: row[1] = int(self.ix[row[1]]) - 1
                elif row[0] == K.OP_U: row[1] = int(self.iu[row[1]]) - 1
            d.update(inds=prog.ravel())
        else:
            raise ArgumentError(f"IndexedConstraint: unsupported constraint {type(con).__name__}")
        return d


def change_dimension(obj, n, m, ix=None, iu=None):
    """``change_dimension(con | cons | cost, n, m, ix, iu)``: the same constraint / ConstraintList / cost acting on ``x[ix]``, ``u[iu]`` of a
    larger model (src/constraints.jl:934-936 and the per-type methods, src/constraint_list.jl:208-217, src/cost_functions.jl:391-401,
    src/lie_costs.jl:144-159)."""
    if isinstance(obj, ConstraintList):
        new = ConstraintList(n, m, obj.N)
        for inds, con in obj.zip():
            add_constraint(new, change_dimension(con, n, m, ix, iu), inds)
        return new
    if isinstance(obj, AbstractConstraint):
        return IndexedConstraint(n, m, obj, ix, iu)
    if isinstance(obj, DiagonalCost):
        ixv, iuv = _index_vec(ix, obj.state_dim), _index_vec(iu, obj.control_dim)
        Qd, Rd, q, r = np.zeros(n), np.zeros(m), np.zeros(n), np.zeros(m)
        Qd[ixv - 1], Rd[iuv - 1], q[ixv - 1], r[iuv - 1] = np.diag(obj.Q), np.diag(obj.R), obj.q, obj.r
        if isinstance(obj, DiagonalQuatCost):
            return DiagonalQuatCost(Qd, Rd, q=q, r=r, c=obj.c, w=obj.w, q_ref=obj.q_ref, q_ind=ixv[obj.q_ind - 1], terminal=obj.terminal)
        return DiagonalCost(Qd, Rd, q=q, r=r, c=obj.c, terminal=obj.terminal)
    raise ArgumentError(f"change_dimension is not defined for {type(obj).__name__}")


class StateBound(BoundConstraint):   # src/constraints.jl:596-617 -- a BoundConstraint whose control block is unbounded
    """``StateBound(n; x_min, x_max)``. The control dimension is taken from the ConstraintList it is added to."""

    def __init__(self, n, x_min=-np.inf, x_max=np.inf):
        self.n = n
        self.x_max, self.x_min = _check_bounds(n, x_max, x_min)
        self.p = int(np.isfinite(self.x_max).sum() + np.isfinite(self.x_min).sum())
        self._bind(0)

    def _bind(self, m):
        self.z_max = np.concatenate([self.x_max, np.full(m, np.inf)]); self.z_min = np.concatenate([self.x_min, np.full(m, -np.inf)])


class ControlBound(BoundConstraint):   # src/constraints.jl:619-640
    """``ControlBound(m; u_min, u_max)``. The state dimension is taken from the ConstraintList it is added to."""

    def __init__(self, m, u_min=-np.inf, u_max=np.inf):
        self.m = m
        self.u_max, self.u_min = _check_bounds(m, u_max, u_min)
        self.p = int(np.isfinite(self.u_max).sum() + np.isfinite(self.u_min).sum())
        self._bind(0)

    def _bind(self, n):
        self.z_max = np.concatenate([np.full(n, np.inf), self.u_max]); self.z_min = np.concatenate([np.full(n, -np.inf), self.u_min])


class ConstraintList:
    """``ConstraintList(n, m, N)``, ``ConstraintList(nx, nu)`` (per-knot dimensions) or ``ConstraintList(models)`` (src/constraint_list.jl:25-66)."""

    def __init__(self, *args):
        if len(args) == 3:
            n, m, N = (int(a) for a in args)
            self.nx, self.nu = [n] * N, [m] * N
        elif len(args) == 2:
            self.nx, self.nu = [int(a) for a in args[0]], [int(a) for a in args[1]]
            if len(self.nx) != len(self.nu):
                raise DimensionMismatch("nx and nu must have one entry per knot point")
        elif len(args) == 1:
            self.nx, self.nu = model_dims(args[0])
        else:
            raise ArgumentError("ConstraintList(n, m, N) | ConstraintList(nx, nu) | ConstraintList(models)")
        self.N = len(self.nx)
        self.n, self.m = self.nx[0], self.nu[0]
        self.constraints, self.inds = [], []
        self.p = np.zeros(self.N, dtype=int)

    uniform = property(lambda s: len(set(s.nx)) == 1 and len(set(s.nu)) == 1)

    def __len__(self):
        return len(self.constraints)

    def __getitem__(self, i):
        return self.constraints[i]

    def __iter__(self):
        return iter(self.constraints)

    def zip(self):   # Base.zip(cons)  src/constraint_list.jl:147
        return zip(self.inds, self.constraints)

    def copy(self):   # Base.copy(cons)  src/constraint_list.jl:54-60: a new list over the same constraint objects
        new = ConstraintList(self.nx, self.nu)
        new.constraints, new.inds, new.p = list(self.constraints), list(self.inds), self.p.copy()
        return new


def add_constraint(cons, con, inds, idx=-1):
    """``add_constraint!(cons, con, inds)`` (src/constraint_list.jl:103-134); ``inds`` = knot ``k`` or ``(first, last)``."""
    first, last = (inds, inds) if np.ndim(inds) == 0 else (inds[0], inds[-1])
    if not (1 <= first <= last <= cons.N):
        raise ArgumentError("Invalid inds, inds[end] must be less than number of knotpoints")   # @assert :107
    for k in range(first, last + 1):     # check_dims at every knot of the range  src/constraint_list.jl:107-111
        nk, mk = cons.nx[k - 1], cons.nu[k - 1]
        if not (getattr(con, "n", nk) == nk and getattr(con, "m", mk) == mk):
            raise DimensionMismatch(f"New constraint not consistent with n={nk} and m={mk} at time step {k}.")
    if isinstance(con, StateBound): con._bind(cons.nu[first - 1])
    if isinstance(con, ControlBound): con._bind(cons.nx[first - 1])
    pos = len(cons.constraints) if idx == -1 else idx
    cons.constraints.insert(pos, con)
    cons.inds.insert(pos, (int(first), int(last)))
    cons.p[first - 1:last] += con.p   # num_constraints!  src/constraint_list.jl:198-206
    cons._version = getattr(cons, "_version", 0) + 1      # see Problem._ensure_current


def num_constraints(cons_or_prob):
    cons = cons_or_prob.constraints if isinstance(cons_or_prob, Problem) else cons_or_prob
    return cons.p.copy()


# ------------------------------------------------------------------------------------------------------------
# Problem (reference src/problem.jl)


class Problem:
    """``Problem(model, obj, x0, tf; xf, constraints, t0, X0, U0, dt)`` (src/problem.jl:79-123) for a batch.

    ``x0`` is ``[n]`` (shared) or ``[B, n]``; ``batch`` gives ``B`` when ``x0`` is shared.  The integrator is RK4
    (the reference's default, src/problem.jl:119-123).  States start as NaN and controls as zeros like the
    reference (src/problem.jl:83-84).  ``error_state=True`` makes the solver kernels (backward / forward pass) work on the
    Lie-group error state of the model (``RD.errstate_dim(model)`` dimensions, Quadrotor: 12) as Altro does for ``LieGroupModel``s.
    """

    def __init__(self, model, obj, *args, xf=None, constraints=None, t0=0.0, X0=None, U0=None, dt=None, batch=None, device=0,
                 error_state=False, **kwargs):
        if "x0" in kwargs:   # src/problem.jl:87-91
            raise ArgumentError("Cannot pass x0 as a keyword argument. It is now a positional argument, and xf is a keyword argument.")
        if kwargs:
            raise ArgumentError(f"unknown keyword arguments {sorted(kwargs)}")
        if len(args) != 2:
            raise ArgumentError("Problem(model, obj, x0, tf; xf, constraints, ...) takes x0 and tf positionally")
        x0, tf = args
        N = len(obj)
        x0 = np.asarray(x0, dtype=float)
        if isinstance(model, AutodiffDynamics):
            # one user model (RD.@autodiff struct M <: ContinuousDynamics + Problem(model, obj, x0, tf)) steps every knot: it is the model
            # vector [model] * (N - 1), on the padded (4, 2) layout the recorded-program kernels exist for
            model = [model] * (N - 1)
        self.hybrid = isinstance(model, (list, tuple))
        if self.hybrid:
            # Problem(models::Vector{<:DiscreteDynamics}, obj, x0, tf)  src/problem.jl:36-73: per-knot dimensions from RD.dims(models); the
            # device works on the padded dimensions (n, m) = (4, 2) with the knot's own entries first (include/trajopt_b200.h to_spec.nx)
            models = list(model)
            nxv, nuv = model_dims(models)                       # DimensionMismatch "Model mismatch at time step k"
            if len(models) != N - 1:
                raise DimensionMismatch("need one model per time step (N - 1 models)")     # @assert length(models) == N-1
            if any(not isinstance(mdl, AutodiffDynamics) for mdl in models):
                raise ArgumentError("a model vector holds AutodiffDynamics models")
            if max(nxv) > 4 or max(nuv) > 2:
                raise ArgumentError("hybrid problems: at most 4 states and 2 controls per knot (the padded kernel instance)")
            n, m = 4, 2
            if error_state:
                raise ArgumentError("error_state=True needs a Lie-group model (RD.errstate_dim(model) != state_dim)")
            if x0.shape[-1] != nxv[0]:
                raise DimensionMismatch("x0 does not match the first model's state dimension")   # @assert length(x0) == nx[1]
            cons = constraints if constraints is not None else ConstraintList(nxv, nuv)
            if cons.nx != nxv:
                raise DimensionMismatch("Constraint state dimensions don't match model")      # src/problem.jl:62
            if cons.nu != nuv:
                raise DimensionMismatch("Constraint control dimensions don't match model")    # src/problem.jl:63
            onx, onu = obj.dims_all()
            if onx != nxv:
                raise DimensionMismatch("Objective state dimensions don't match model.")      # src/problem.jl:65
            if onu != nuv:
                raise DimensionMismatch("Objective control dimensions don't match model.")    # src/problem.jl:66
            x0 = np.concatenate([x0, np.zeros(x0.shape[:-1] + (n - nxv[0],))], axis=-1)
            self.nx, self.nu = nxv, nuv
            nf = nxv[-1]
        else:
            n, m = model.dims()
            if x0.shape[-1] != n:
                raise DimensionMismatch("x0 does not match the model's state dimension")   # @assert src/problem.jl:48
            onx, onu = obj.dims_all()
            if any(a != n for a in onx):
                raise DimensionMismatch("Objective state dimensions don't match model.")      # src/problem.jl:67
            if any(a != m for a in onu):
                raise DimensionMismatch("Objective control dimensions don't match model.")    # src/problem.jl:68
            cons = constraints if constraints is not None else ConstraintList(n, m, N)
            if any(a != n for a in cons.nx) or any(a != m for a in cons.nu):
                raise DimensionMismatch("Constraint state dimensions don't match model")   # src/problem.jl:64-65
            self.nx, self.nu = [n] * N, [m] * N
            nf = n
        B = int(batch) if batch is not None else (x0.shape[0] if x0.ndim == 2 else 1)
        if cons.N != N:
            raise DimensionMismatch("ConstraintList horizon does not match the objective")
        if dt is None:
            dtv = np.full(N - 1, float(tf - t0) / (N - 1))
        else:
            dtv = np.full(N - 1, float(dt)) if np.ndim(dt) == 0 else np.asarray(dt, dtype=float)
        if not tf > t0:
            raise ArgumentError("tf must be greater than t0")   # @assert tf > t0 src/problem.jl:52
        if dtv.shape != (N - 1,) or not np.isclose(dtv.sum(), tf - t0, rtol=1e-8):
            raise ArgumentError("the time steps must add up to tf - t0")   # @assert in SampledTrajectory(...; tf, dt), test/problems_tests.jl:86
        self.model, self.obj, self.constraints = model, obj, cons
        self.N, self.n, self.m, self.B = N, n, m, B
        if error_state and model.errstate_dim() == n:
            raise ArgumentError("error_state=True needs a Lie-group model (RD.errstate_dim(model) != state_dim)")
        self.error_state = bool(error_state)
        self.ne = model.errstate_dim() if error_state else n
        self.x0 = np.broadcast_to(x0, (B, n)).copy()
        self.xf = np.full(nf, np.nan) if xf is None else np.asarray(xf, dtype=float).copy()
        self._device = device
        self._dt = np.array(dtv, dtype=float)        # the time steps as given: a rebuild must not re-derive them from the knot times
        self.spec = self._make_spec(dtv, t0)
        self._open()
        self._sig = self._signature()
        self._call("to_set_initial_state", K._dp(self.x0))
        if U0 is not None:
            initial_controls(self, U0)
        if X0 is not None:
            initial_states(self, X0)

    def _make_spec(self, dtv, t0):
        """the ABI description of the current host-side problem (cost table, constraint list, models)"""
        cons = self.constraints
        if not self.hybrid:
            uniq, index = self.obj._tables()
            self._cost_objs = uniq
            con_specs = [c._spec(f, l) for (f, l), c in zip(cons.inds, cons.constraints)]
            return K.Spec(self.model.model_id, self.n, self.m, self.N, self.B, dtv, [c._spec() for c in uniq], index, con_specs,
                          params=self.model.params, t0=t0, device=self._device, error_state=self.error_state)
        # hybrid: every cost / constraint is re-expressed on the padded [x(4); u(2)] layout (change_dimension, src/cost_functions.jl:391-401,
        # src/constraints.jl:934-936); the unused controls get a unit weight so that Quu stays positive definite -- they stay exactly zero
        n, m = self.n, self.m
        padded, uniq, index, seen = {}, [], [], {}
        self._cost_objs = []
        for k, c in enumerate(self.obj.cost):
            key = (id(c), self.nx[k], self.nu[k])
            if key not in padded:
                if not isinstance(c, DiagonalCost) or isinstance(c, DiagonalQuatCost):
                    raise ArgumentError("hybrid problems take DiagonalCost / LQRCost stage costs")
                pc = c
                if (self.nx[k], self.nu[k]) != (n, m):
                    nk, mk = self.nx[k], self.nu[k]
                    Qd, Rd, q, r = np.zeros(n), np.ones(m), np.zeros(n), np.zeros(m)
                    Qd[:nk], Rd[:mk], q[:nk], r[:mk] = np.diag(c.Q), np.diag(c.R), c.q, c.r
                    pc = DiagonalCost(Qd, Rd, q=q, r=r, c=c.c, terminal=c.terminal, checks=False)
                padded[key] = pc
                seen[key] = len(uniq); uniq.append(pc); self._cost_objs.append(c)
            index.append(seen[key])
        con_specs = []
        for (f, l), c in zip(cons.inds, cons.constraints):
            nk, mk = self.nx[f - 1], self.nu[f - 1]
            pc = c if (nk, mk) == (n, m) else IndexedConstraint(n, m, c, (1, nk), (1, mk))
            con_specs.append(pc._spec(f, l))
        mods, dyn_index, mseen = [], [], {}
        for mdl in self.model:
            if id(mdl) not in mseen:
                mseen[id(mdl)] = len(mods); mods.append(mdl._spec())
            dyn_index.append(mseen[id(mdl)])
        return K.Spec(K.MODEL_EXPR, n, m, self.N, self.B, dtv, [c._spec() for c in uniq], index, con_specs, t0=t0, device=self._device,
                      dyn=mods, dyn_index=dyn_index, nx=self.nx, nu=self.nu)

    def _open(self):
        """create the device-side problem (to_create); fails loudly without the CUDA library / a GPU."""
        self._lib = K.load_library()
        self._h = C.c_void_p()
        rc = self._lib.to_create(C.byref(self.spec.c), C.byref(self._h))
        K.check(self._lib, None, rc)

    def _signature(self):
        """what the device-side tables were built from: the cost object of every knot, the constraint list, and the version counters the
        mutating helpers of the reference API bump (set_LQR_goal!(prob.obj[k], ...), add_constraint!(get_constraints(prob), ...))"""
        cons = self.constraints
        return (tuple(id(c) for c in self.obj.cost), tuple(getattr(c, "_version", 0) for c in self._cost_objs),
                tuple(id(c) for c in cons.constraints), tuple(cons.inds), getattr(cons, "_version", 0))

    def _ensure_current(self):
        """The reference mutates a live problem's objective / constraint list in place.  The device tables are a copy taken at
        construction, so a change is re-uploaded here, before the next device call: the handle is rebuilt from the current host
        description with the live trajectory, initial state and solver options carried over (multipliers and penalties restart,
        as they must when the constraint list changes shape)."""
        if getattr(self, "_sig", None) is None or self._sig == self._signature():
            return
        X, U = np.empty((self.B, self.N, self.n)), np.empty((self.B, self.N - 1, self.m))
        self._raw_call("to_get_states", K._dp(X)); self._raw_call("to_get_controls", K._dp(U))
        t = np.empty(self.N)
        self._raw_call("to_get_times", K._dp(t))
        opts = getattr(self, "_options", None)
        # Per-instance state is carried over row by row.  The later change wins: a cost mutated since the handle was built, or a Goal
        # constraint whose xf changed since the per-instance call, takes its new (shared) value in every instance; a constraint added
        # since keeps the value it was built with.
        carry = {}
        if getattr(self, "_inst", False):
            q, r = np.empty((self.B, len(self._cost_objs), self.n)), np.empty((self.B, len(self._cost_objs), self.m))
            self._raw_call("to_get_cost_terms", K._dp(q), K._dp(r))
            built = self._sig[1]
            carry = {id(c): (q[:, j].copy(), r[:, j].copy()) for j, c in enumerate(self._cost_objs) if getattr(c, "_version", 0) == built[j]}
        con_carry = {}   # per-instance constraint rows (Goal values, constraint data): those of every constraint unchanged since the call
        snap = getattr(self, "_con_snap", {})
        live = {id(c): c for c in self.constraints.constraints}
        for j, cid in enumerate(self._sig[2]):
            con = live.get(cid)
            if cid in snap and con is not None and np.array_equal(_con_snap_row(con), snap[cid]):
                rows = np.empty((self.B, snap[cid].size))
                self._raw_call(_con_rows_call(con, "get"), j, K._dp(rows))
                con_carry[cid] = rows
        mparams = None
        if getattr(self, "_mparams", False):   # per-instance model parameters: carried over as they are
            mparams = np.empty((self.B, len(self.model.params)))
            self._raw_call("to_get_model_params", K._dp(mparams))
        self.close()
        self.spec = self._make_spec(self._dt, float(t[0]))
        self._open()
        self._sig = self._signature()
        self._inst = bool(carry)
        if carry:
            q, r = np.empty((self.B, len(self._cost_objs), self.n)), np.empty((self.B, len(self._cost_objs), self.m))
            self._raw_call("to_get_cost_terms", K._dp(q), K._dp(r))
            for j, c in enumerate(self._cost_objs):
                if id(c) in carry:
                    q[:, j], r[:, j] = carry[id(c)]
            self._raw_call("to_set_cost_terms", K._dp(q), K._dp(r))
        for j, c in enumerate(self.constraints.constraints):
            if id(c) in con_carry:
                self._raw_call(_con_rows_call(c, "set"), j, K._dp(con_carry[id(c)]))
        self._con_snap = {cid: v for cid, v in snap.items() if cid in con_carry}
        if mparams is not None:
            self._raw_call("to_set_model_params", K._dp(mparams), int(mparams.shape[1]))
        self._raw_call("to_set_initial_state", K._dp(self.x0))
        self._raw_call("to_set_controls", K._dp(U))
        if np.all(np.isfinite(X)):
            self._raw_call("to_set_states", K._dp(X))
        if opts is not None:
            self._raw_call("to_set_options", C.byref(opts))

    def _call(self, name, *args):
        self._ensure_current()
        self._raw_call(name, *args)

    def _raw_call(self, name, *args):
        rc = getattr(self._lib, name)(self._h, *args)
        K.check(self._lib, self._h, rc)

    def _default_options(self, o):
        self._lib.to_default_options(C.byref(o))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.to_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def dims(prob, k=None):   # RD.dims(prob) / RD.dims(prob, k)  src/problem.jl:146-147 ; RD.dims(models)  src/dynamics.jl:15 ; RD.dims(obj)
    if isinstance(prob, (list, tuple)):
        return model_dims(prob)
    if isinstance(prob, Objective):
        return prob.dims_all()
    if k is not None:
        return prob.nx[k - 1], prob.nu[k - 1], prob.N
    if getattr(prob, "hybrid", False):
        return list(prob.nx), list(prob.nu), prob.N
    return prob.n, prob.m, prob.N


def state_dim(obj, k=1):   # RD.state_dim(prob | obj, k), state_dim(cost | con)  src/problem.jl:149, src/objective.jl:60
    if isinstance(obj, Objective): return obj[k - 1].state_dim
    if isinstance(obj, Problem): return obj.nx[k - 1]
    return obj.state_dim if isinstance(obj, CostFunction) else obj.n


def control_dim(obj, k=1):   # RD.control_dim(prob | obj, k)  src/problem.jl:150, src/objective.jl:61
    if isinstance(obj, Objective): return obj[k - 1].control_dim
    if isinstance(obj, Problem): return obj.nu[k - 1]
    return obj.control_dim if isinstance(obj, CostFunction) else obj.m


def get_J(obj):   # get_J(obj)  src/objective.jl:110: the per-knot cost scratch of an objective (filled by cost_knots for instance 0)
    return obj.J


def get_initial_time(prob):   # src/problem.jl:189
    return float(gettimes(prob)[0])


def get_final_time(prob):   # src/problem.jl:196
    return float(gettimes(prob)[-1])


def get_trajectory(prob):
    """``get_trajectory(prob)`` (src/problem.jl:222): the sampled trajectory as ``(X[B, N, n], U[B, N-1, m], t[N])``."""
    return states(prob), controls(prob), gettimes(prob)


def initial_trajectory(prob, X0, U0):   # initial_trajectory!(prob, Z0)  src/problem.jl:242-245
    initial_states(prob, X0)
    initial_controls(prob, U0)


def copy_problem(prob, cls=None, **overrides):
    """``copy(prob)`` / ``Problem(p; model, obj, constraints, x0, xf, t0, tf)`` (src/problem.jl:125-128, :342-345): a new batch with copies of
    the objective and the constraint list (the constraint objects themselves are shared, as ``copy(::ConstraintList)`` does), the same x0, xf,
    time grid and the current trajectory."""
    t = gettimes(prob)
    obj = overrides.pop("obj", prob.obj.copy())
    cons = overrides.pop("constraints", prob.constraints.copy())
    new = (cls or type(prob))(overrides.pop("model", prob.model), obj, overrides.pop("x0", prob.x0.copy()), float(t[-1]),
                              xf=overrides.pop("xf", prob.xf.copy()), constraints=cons, t0=float(t[0]), dt=np.diff(t),
                              error_state=prob.error_state, **overrides)
    X, U = states(prob), controls(prob)
    if np.all(np.isfinite(X)):
        initial_states(new, X)
    initial_controls(new, U)
    return new


def horizonlength(prob):
    return prob.N


def get_model(prob):
    return prob.model


def get_objective(prob):
    return prob.obj


def get_constraints(prob):
    return prob.constraints


def get_initial_state(prob):
    return prob.x0


def get_final_state(prob):
    return prob.xf


def is_constrained(prob):
    """True when the problem has constraints.  (The reference returns ``isempty(constraints)``, an inverted
    test enshrined in test/problems_tests.jl:208 -- SURVEY.md 2.4; this mirror returns the intended value.)"""
    return len(prob.constraints) > 0


def _bcast(a, shape, what):
    a = np.asarray(a, dtype=np.float64)
    try:
        return np.ascontiguousarray(np.broadcast_to(a, shape))
    except ValueError:
        raise DimensionMismatch(f"{what} has shape {a.shape}, expected broadcastable to {shape}")


def initial_controls(prob, U0):   # initial_controls!  src/problem.jl:261
    U = _bcast(U0, (prob.B, prob.N - 1, prob.m), "U0")
    prob._call("to_set_controls", K._dp(U))


def initial_states(prob, X0):   # initial_states!  src/problem.jl:253
    X = _bcast(X0, (prob.B, prob.N, prob.n), "X0")
    prob._call("to_set_states", K._dp(X))


def set_initial_state(prob, x0):   # set_initial_state!  src/problem.jl:270
    prob.x0 = _bcast(x0, (prob.B, prob.n), "x0").copy()
    prob._call("to_set_initial_state", K._dp(prob.x0))


def setinitialtime(prob, t0):   # RD.setinitialtime!  src/problem.jl:280
    tf = C.c_double()
    prob._call("to_set_initial_time", float(t0), C.byref(tf))
    return tf.value


def set_goal_state(prob, xf, objective=True, constraint=True):   # set_goal_state!  src/problem.jl:294-310
    """``xf[n]``: the goal of every instance.  ``xf[B, n]``: instance ``b`` goes to ``xf[b]`` (``set_goal_state!`` per instance: its own
    linear cost terms ``q = -Q xf[b]`` and Goal constraint values; the shared cost / constraint objects are left as they are)."""
    xf = np.ascontiguousarray(np.asarray(xf, dtype=np.float64))
    if xf.ndim == 2:
        if xf.shape != (prob.B, prob.n):
            raise DimensionMismatch(f"set_goal_state!: xf has shape {xf.shape}, expected ({prob.n},) or ({prob.B}, {prob.n})")
        prob._call("to_set_goal_states", K._dp(xf), int(objective), int(constraint))
        if objective:
            prob._inst = True
        if constraint:   # the Goal constraints that now hold per-instance values, with the xf they had (a later change to it wins)
            prob._con_snap = {**getattr(prob, "_con_snap", {}),
                              **{id(c): _con_snap_row(c) for c in prob.constraints if isinstance(c, GoalConstraint)}}
        prob.xf = xf.copy()
        return
    if objective:
        for c in prob._cost_objs:
            if isinstance(c, QuadraticCostFunction):
                set_LQR_goal(c, xf)
    if constraint:
        for con in prob.constraints:
            if isinstance(con, GoalConstraint):
                con.xf = xf[con.inds - 1].copy() if xf.size != con.xf.size else xf.copy()
    prob.xf = xf.copy()
    if constraint:   # every instance takes the shared Goal values
        goals = {id(c) for c in prob.constraints if isinstance(c, GoalConstraint)}
        prob._con_snap = {cid: v for cid, v in getattr(prob, "_con_snap", {}).items() if cid not in goals}
    prob._call("to_set_goal_state", K._dp(xf), int(objective), int(constraint))


def update_trajectory(prob, Xref, Uref, start=1):
    """``update_trajectory!(obj, Z, start)`` (src/objective.jl:198-212): knot ``i`` of the problem's (tracking) objective follows
    row ``start - 1 + i`` of the reference ``Xref[nref, n]``, ``Uref[nref, m]`` -- ``set_LQR_goal!`` on every knot's cost.
    ``Xref[B, nref, n]``, ``Uref[B, nref, m]``: instance ``b`` tracks its own reference (same ``start``); the shared cost objects
    are left as they are."""
    Xref = np.ascontiguousarray(np.asarray(Xref, dtype=np.float64)); Uref = np.ascontiguousarray(np.asarray(Uref, dtype=np.float64))
    if Xref.ndim == 3 or Uref.ndim == 3:
        if (Xref.ndim != 3 or Uref.ndim != 3 or Xref.shape[0] != prob.B or Uref.shape[0] != prob.B or Xref.shape[2] != prob.n
                or Uref.shape[2] != prob.m or Uref.shape[1] != Xref.shape[1]):
            raise DimensionMismatch("update_trajectory!: per-instance Xref must be [B, nref, n] and Uref [B, nref, m]")
        if start < 1 or start - 1 + prob.N > Xref.shape[1]:
            raise DimensionMismatch("update_trajectory!: the reference is shorter than start + N - 1")
        if not all(isinstance(c, QuadraticCostFunction) for c in prob.obj):
            raise ArgumentError("update_trajectory! is defined for objectives of QuadraticCostFunctions (src/objective.jl:207)")
        prob._call("to_update_trajectories", K._dp(Xref), K._dp(Uref), int(Xref.shape[1]), int(start))
        prob._inst = True
        return
    if Xref.ndim != 2 or Uref.ndim != 2 or Xref.shape[1] != prob.n or Uref.shape[1] != prob.m or Uref.shape[0] != Xref.shape[0]:
        raise DimensionMismatch("update_trajectory!: Xref must be [nref, n] and Uref [nref, m]")
    if start < 1 or start - 1 + prob.N > Xref.shape[0]:
        raise DimensionMismatch("update_trajectory!: the reference is shorter than start + N - 1")
    if not all(isinstance(c, QuadraticCostFunction) for c in prob.obj):
        raise ArgumentError("update_trajectory! is defined for objectives of QuadraticCostFunctions (src/objective.jl:207)")
    for i, k in enumerate(range(start - 1, start - 1 + prob.N)):
        set_LQR_goal(prob.obj[i], Xref[k], Uref[k])
    prob._call("to_update_trajectory", K._dp(Xref), K._dp(Uref), int(Xref.shape[0]), int(start))


def cost_terms(prob):
    """The linear terms of every distinct cost of every instance: ``q[B, ncost, n]``, ``r[B, ncost, m]`` (the shared ones broadcast when no
    per-instance goal was set).  ``ncost`` counts the distinct cost objects of the objective, in order of first use."""
    nc = len(prob._cost_objs)
    q, r = np.empty((prob.B, nc, prob.n)), np.empty((prob.B, nc, prob.m))
    prob._call("to_get_cost_terms", K._dp(q), K._dp(r))
    return q, r


def set_cost_terms(prob, q, r):
    """``set_LQR_goal!(obj[k], ...)`` per instance with raw terms: ``q[B, ncost, n]``, ``r[B, ncost, m]`` (layout of ``cost_terms``)."""
    nc = len(prob._cost_objs)
    q = np.ascontiguousarray(np.asarray(q, dtype=np.float64)); r = np.ascontiguousarray(np.asarray(r, dtype=np.float64))
    if q.shape != (prob.B, nc, prob.n) or r.shape != (prob.B, nc, prob.m):
        raise DimensionMismatch(f"set_cost_terms: expected q [{prob.B}, {nc}, {prob.n}] and r [{prob.B}, {nc}, {prob.m}], got {q.shape} and {r.shape}")
    prob._ensure_current()
    if len(prob._cost_objs) != nc:
        raise DimensionMismatch("set_cost_terms: the objective changed its distinct costs; read cost_terms again")
    prob._call("to_set_cost_terms", K._dp(q), K._dp(r))
    prob._inst = True


def _model_param_rows(prob, params):
    """``params`` as the ``[B, nparams]`` rows ``to_set_model_params`` takes; every check that needs no device happens here"""
    if getattr(prob, "hybrid", False):
        raise ArgumentError("per-instance model parameters are not supported on hybrid problems (their constants live in the recorded programs)")
    nparams = len(prob.model.params)
    if isinstance(params, (list, tuple)) and any(isinstance(x, _Model) for x in params):
        if len(params) != prob.B:
            raise DimensionMismatch(f"set_model_params: {len(params)} models for a batch of {prob.B} instances")
        for b, x in enumerate(params):
            if type(x) is not type(prob.model) or x.dims() != prob.model.dims():
                raise ArgumentError(f"set_model_params: instance {b} holds a {type(x).__name__} {getattr(x, 'dims', lambda: '')()}, the problem's model is "
                                    f"a {type(prob.model).__name__} {prob.model.dims()}")
        params = [x.params for x in params]
    rows = np.ascontiguousarray(np.asarray(params, dtype=np.float64))
    if rows.shape != (prob.B, nparams):
        raise DimensionMismatch(f"set_model_params: expected [{prob.B}, {nparams}] parameters, got {rows.shape}")
    return rows


def set_model_params(prob, params):
    """Instance ``b`` integrates its dynamics with its own model parameters: ``params[B, nparams]`` in the order of ``model.params``, or a
    sequence of ``B`` models of ``type(prob.model)`` whose ``.params`` are taken.  A batch with per-instance parameters computes, bit for bit,
    what each instance computes in a batch built with its model.  The trajectory is not rolled out again; the next rollout, expansion, line
    search or solve uses the new values.  ``prob.model`` is left as it is."""
    rows = _model_param_rows(prob, params)
    prob._call("to_set_model_params", K._dp(rows), int(rows.shape[1]))
    prob._mparams = True


def model_params(prob):
    """The model parameters of every instance, ``[B, nparams]`` (the shared ``model.params`` broadcast when none were set)."""
    if getattr(prob, "hybrid", False):
        raise ArgumentError("hybrid problems have no model parameter vector")
    out = np.empty((prob.B, len(prob.model.params)))
    prob._call("to_get_model_params", K._dp(out))
    return out


# which fields of a constraint's _spec are its per-instance data, in the order of an instance's row (include/trajopt_b200.h
# to_set_constraint_data); every other field stays shared
_CON_DATA_FIELDS = {K.CON_BOUND: ("a", "b"), K.CON_LINEAR: ("b",), K.CON_CIRCLE: ("a", "b", "rad"), K.CON_SPHERE: ("a", "b", "c", "rad"),
                    K.CON_NORM: ("val",), K.CON_COLLISION: ("val",)}


def _con_row(con):
    """(spec, row): the device description of ``con`` and its data in the layout of one instance's row (ArgumentError: no such data)"""
    if isinstance(con, (QuatVecEq, AutodiffConstraint, IndexedConstraint)):
        raise ArgumentError(f"the data of a {type(con).__name__} stays shared across the batch")
    spec = con._spec(1, 1)
    fields = _CON_DATA_FIELDS.get(spec["kind"])
    if fields is None:
        raise ArgumentError(f"{type(con).__name__} carries no per-instance constraint data")
    return spec, np.concatenate([np.atleast_1d(np.asarray(spec[f], dtype=np.float64)).ravel() for f in fields])


def _con_snap_row(con):
    """the row ``con`` holds in every instance until a per-instance call: a Goal's ``xf``, another kind's data (``_con_row``)"""
    return np.array(con.xf, dtype=float) if isinstance(con, GoalConstraint) else _con_row(con)[1]


def _con_rows_call(con, verb):
    """the C call that sets (``verb = "set"``) or reads (``"get"``) the per-instance rows of ``con``: a Goal's values or another kind's data"""
    return f"to_{verb}_goal_values" if isinstance(con, GoalConstraint) else f"to_{verb}_constraint_data"


def _con_and_index(prob, con):
    """(index, constraint) of ``con``: an index into the problem's constraint list or one of its constraint objects"""
    j = _con_index(prob, con)
    if not 0 <= j < len(prob.constraints):
        raise ArgumentError(f"constraint index {j} outside 0:{len(prob.constraints) - 1}")
    return j, prob.constraints[j]


def _constraint_data_rows(prob, con, rows):
    """(index, constraint, rows [B, len]) as to_set_constraint_data / to_set_goal_values take them; every check that needs no device happens here"""
    if getattr(prob, "hybrid", False):
        raise ArgumentError("per-instance constraint data is not supported on hybrid problems")
    j, con = _con_and_index(prob, con)
    objs = isinstance(rows, (list, tuple)) and any(isinstance(x, AbstractConstraint) for x in rows)
    if isinstance(con, GoalConstraint):
        if objs:
            if len(rows) != prob.B:
                raise DimensionMismatch(f"set_constraint_data: {len(rows)} constraints for a batch of {prob.B} instances")
            if any(type(x) is not GoalConstraint or not np.array_equal(x.inds, con.inds) for x in rows):
                raise ArgumentError("set_constraint_data: every instance's constraint must be a GoalConstraint on the same indices")
            rows = [x.xf for x in rows]
        out = np.ascontiguousarray(np.asarray(rows, dtype=np.float64))
        if out.shape != (prob.B, con.p):
            raise DimensionMismatch(f"set_constraint_data: expected [{prob.B}, {con.p}] Goal values, got {out.shape}")
        return j, con, out
    spec, shared = _con_row(con)
    if objs:
        if len(rows) != prob.B:
            raise DimensionMismatch(f"set_constraint_data: {len(rows)} constraints for a batch of {prob.B} instances")
        fields = _CON_DATA_FIELDS[spec["kind"]]
        packed = []
        for b, x in enumerate(rows):
            if type(x) is not type(con):
                raise ArgumentError(f"set_constraint_data: instance {b} holds a {type(x).__name__}, the constraint is a {type(con).__name__}")
            xs, xr = _con_row(x)
            same = all(np.array_equal(np.asarray(xs[k]), np.asarray(spec[k])) for k in spec if k not in fields and k in xs) and set(xs) == set(spec)
            if xr.shape != shared.shape or not same:
                raise DimensionMismatch(f"set_constraint_data: instance {b}'s {type(x).__name__} differs from the problem's in more than its data")
            packed.append(xr)
        rows = packed
    out = np.ascontiguousarray(np.asarray(rows, dtype=np.float64))
    if out.shape != (prob.B, shared.size):
        raise DimensionMismatch(f"set_constraint_data: expected [{prob.B}, {shared.size}] rows, got {out.shape}")
    for b in range(prob.B):
        r = out[b]
        if spec["kind"] == K.CON_BOUND:
            nm = shared.size // 2
            fin = np.isfinite(shared)
            bad = np.nonzero(np.where(fin, ~np.isfinite(r), r != shared))[0]
            if bad.size:
                raise ArgumentError(f"set_constraint_data: instance {b}, entry {bad[0]}: BoundConstraint entries must be finite exactly where the "
                                    "shared bound is, with the same infinities")
            bad = np.nonzero(~(r[:nm] >= r[nm:]))[0]
            if bad.size:
                raise ArgumentError(f"set_constraint_data: instance {b}, entry {bad[0]}: Upper bounds must be greater than or equal to lower bounds")
        else:
            bad = np.nonzero(~np.isfinite(r))[0]
            if bad.size:
                raise ArgumentError(f"set_constraint_data: instance {b}, entry {bad[0]} is not finite")
            if spec["kind"] == K.CON_NORM and not r[0] >= 0:
                raise ArgumentError(f"set_constraint_data: instance {b}: NormConstraint value must be non-negative")
    return j, con, out


def set_constraint_data(prob, con, rows):
    """Instance ``b`` evaluates constraint ``con`` (an index into the problem's constraint list, or the constraint object) with its own data.
    ``rows`` is ``[B, len]`` in the layout of include/trajopt_b200.h (BoundConstraint ``z_max | z_min``, LinearConstraint ``b``,
    CircleConstraint ``xc | yc | r``, SphereConstraint ``xc | yc | zc | r``, NormConstraint ``val``, CollisionConstraint ``radius``;
    GoalConstraint ``xf[inds]``), or a sequence of ``B`` constraints of the same type and shape whose data are taken.  A batch whose
    instance ``b`` holds ``d_b`` computes, bit for bit, what instance ``b`` of a batch built with ``d_b`` computes.  The constraint objects
    are left as they are; a later in-place change to one of them, picked up when the handle is rebuilt, wins in every instance.
    An ``IndexedConstraint`` (a constraint applied to a slice of a larger model) keeps its data shared: ``ArgumentError``."""
    j, con, out = _constraint_data_rows(prob, con, rows)
    prob._call(_con_rows_call(con, "set"), j, K._dp(out))
    prob._con_snap = {**getattr(prob, "_con_snap", {}), id(con): _con_snap_row(con)}


def constraint_data(prob, con):
    """The data of constraint ``con`` of every instance, ``[B, len]`` (the shared data broadcast when none was set)."""
    j, con = _con_and_index(prob, con)
    out = np.empty((prob.B, _con_snap_row(con).size))
    prob._call(_con_rows_call(con, "get"), j, K._dp(out))
    return out


def shift_trajectory(prob, steps=1):
    """Receding-horizon warm start on the device (no reference counterpart: MPC user code around Altro does this on the host):
    ``X_k <- X_{k+steps}``, ``U_k <- U_{k+steps}`` with the tail repeated, multipliers moved with their knots,
    ``x0 <- X_{1+steps}``, ``t0`` advanced.  Follow with ``set_initial_state`` (measured state) and ``rollout``."""
    prob._call("to_shift_trajectory", int(steps))


def states(prob, k=None):   # states(prob)  src/problem.jl:175
    X = np.empty((prob.B, prob.N, prob.n))
    prob._call("to_get_states", K._dp(X))
    return X if k is None else X[:, k - 1]


def controls(prob, k=None):   # controls(prob)  src/problem.jl:168
    U = np.empty((prob.B, prob.N - 1, prob.m))
    prob._call("to_get_controls", K._dp(U))
    return U if k is None else U[:, k - 1]


def gettimes(prob):   # gettimes(prob)  src/problem.jl:182
    t = np.empty(prob.N)
    prob._call("to_get_times", K._dp(t))
    return t


def rollout(prob):   # rollout!(prob)  src/problem.jl:330-340
    prob._call("to_rollout")


def cost(prob):   # cost(prob)  src/problem.jl:321 -> [B]
    J = np.empty(prob.B)
    prob._call("to_cost", K._dp(J))
    return J


def cost_knots(prob):   # cost!(obj, Z); get_J(obj)  src/objective.jl:104-110 -> [B, N]
    Jk = np.empty((prob.B, prob.N))
    prob._call("to_cost_knots", K._dp(Jk))
    prob.obj.J[:] = Jk[0]                      # the reference's shared scratch obj.J (one instance): instance 0 of the batch
    return Jk


def cost_gradient(prob):   # RD.gradient!(cost_k, grad, z_k) for all knots  src/cost_functions.jl:137-172 -> [B, N, n+m]
    g = np.empty((prob.B, prob.N, prob.n + prob.m))
    prob._call("to_cost_gradient", K._dp(g))
    return g


def cost_hessian(prob):   # RD.hessian!  src/cost_functions.jl:212-233 -> [B, N, n+m, n+m]
    nm = prob.n + prob.m
    H = np.empty((prob.B, prob.N, nm, nm))
    prob._call("to_cost_hessian", K._dp(H))
    return np.swapaxes(H, -1, -2)


def _con_index(prob, con):
    if isinstance(con, (int, np.integer)):
        return int(con)
    for i, c in enumerate(prob.constraints):
        if c is con:
            return i
    raise ArgumentError("constraint is not part of the problem's ConstraintList")


def evaluate_constraints(prob, con):
    """``evaluate_constraints!(sig, con, vals, Z, inds)`` (src/abstract_constraint.jl:200-225) -> ``[B, len(inds), p]``."""
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    vals = np.empty((prob.B, last - first + 1, prob.constraints[i].p))
    prob._call("to_eval_constraints", i, K._dp(vals))
    return vals


def constraint_jacobians(prob, con):
    """``constraint_jacobians!`` (src/abstract_constraint.jl:236-248) -> ``[B, len(inds), p, n+m]``."""
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    p = prob.constraints[i].p
    jac = np.empty((prob.B, last - first + 1, prob.n + prob.m, p))
    prob._call("to_constraint_jacobians", i, K._dp(jac))
    return np.swapaxes(jac, -1, -2)


def constraint_hessians(prob, con, lam=None):
    """``∇constraint_jacobians!(sig, diff, con, H, λ, c, Z, inds)`` (src/abstract_constraint.jl:267-280): the second-order constraint term
    ``d/dz (∇c' λ)`` of every knot in the constraint's range -> ``[B, len(inds), n+m, n+m]``; ``lam`` ``[B, len, p]`` (default: the
    problem's current multipliers)."""
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    nm = prob.n + prob.m
    H = np.empty((prob.B, last - first + 1, nm, nm))
    lp = None if lam is None else K._dp(_bcast(lam, (prob.B, last - first + 1, prob.constraints[i].p), "lambda"))
    prob._call("to_constraint_hessians", i, lp, K._dp(H))
    return H


def max_violation(prob):
    v = np.empty(prob.B)
    prob._call("to_max_violation", K._dp(v))
    return v


def merit(prob):
    """cost + augmented-Lagrangian penalty of the current trajectory -> [B]."""
    J = np.empty(prob.B)
    prob._call("to_merit", K._dp(J))
    return J


def al_expansion(prob):
    nm = prob.n + prob.m
    g = np.empty((prob.B, prob.N, nm))
    H = np.empty((prob.B, prob.N, nm, nm))
    prob._call("to_al_expansion", K._dp(g), K._dp(H))
    return g, np.swapaxes(H, -1, -2)


# ---- what Altro.jl does with the API above ---------------------------------------------------------------------


def expand(prob):
    """dynamics expansion (RD.jacobian!(ForwardAD) at every knot)."""
    prob._call("to_expand")


def dynamics_jacobians(prob):
    """-> ``[B, N-1, n, n+m]`` = [A B] per knot."""
    AB = np.empty((prob.B, prob.N - 1, prob.n + prob.m, prob.n))
    prob._call("to_get_dynamics_jacobians", K._dp(AB))
    return np.swapaxes(AB, -1, -2)


def backward(prob):
    status = np.empty(prob.B, dtype=np.int32)
    prob._call("to_backward", K._ip(status))
    return status


def forward(prob):
    J, alpha = np.empty(prob.B), np.empty(prob.B)
    prob._call("to_forward", K._dp(J), K._dp(alpha))
    return J, alpha


def ilqr_step(prob, iters=1):
    prob._call("to_ilqr_step", int(iters))


def al_update(prob):
    prob._call("to_al_update")


def gains(prob):
    """-> ``K[B, N-1, m, n_e]``, ``d[B, N-1, m]`` (``n_e = n`` unless the problem uses the error state)."""
    Kk = np.empty((prob.B, prob.N - 1, prob.ne, prob.m))
    d = np.empty((prob.B, prob.N - 1, prob.m))
    prob._call("to_get_gains", K._dp(Kk), K._dp(d))
    return np.swapaxes(Kk, -1, -2), d


def errstate_dim(prob):
    """``RD.errstate_dim`` as the solver kernels see it: ``n``, or the model's error-state dimension with ``error_state=True``."""
    ne = C.c_int32()
    prob._call("to_error_state_dim", C.byref(ne))
    return ne.value


def state_diff(prob, Xbar):
    """``RD.state_diff(model, xbar_k, x_k)`` of every knot of ``Xbar[B, N, n]`` against the current trajectory -> ``[B, N, n_e]``."""
    Xb = _bcast(Xbar, (prob.B, prob.N, prob.n), "Xbar")
    dx = np.empty((prob.B, prob.N, prob.ne))
    prob._call("to_state_diff", K._dp(Xb), K._dp(dx))
    return dx


def error_dynamics(prob):
    """error-state dynamics Jacobians ``[A_e B_e] = G_{k+1}' [A G_k | B]`` -> ``[B, N-1, n_e, n_e+m]`` (after ``expand``)."""
    AB = np.empty((prob.B, prob.N - 1, prob.ne + prob.m, prob.ne))
    prob._call("to_get_error_dynamics", K._dp(AB))
    return np.swapaxes(AB, -1, -2)


def error_expansion(prob):
    """cost + AL expansion in the error state (Altro ``error_expansion!``) -> ``grad[B, N, n_e+m]``, ``hess[B, N, n_e+m, n_e+m]``."""
    nm = prob.ne + prob.m
    g = np.empty((prob.B, prob.N, nm))
    H = np.empty((prob.B, prob.N, nm, nm))
    prob._call("to_error_expansion", K._dp(g), K._dp(H))
    return g, np.swapaxes(H, -1, -2)


def expansion_records(prob):
    """Diagnostic, CUDA problems on the record path only (``backward_algebra(prob) == 1``): the cost + AL expansion that the last backward
    pass read from the per-knot records -> ``[B, N, 48]`` = ``g~[16] | hd[16] | Hb[4, 4]`` in the physical order of csrc/frag_layout.cuh."""
    out = np.empty((prob.B, prob.N, 48))
    prob._call("to_get_expansion_records", K._dp(out))
    return out


def errstate_jacobian(prob):
    """``RD.errstate_jacobian!(model, G, z)`` of every knot of the current trajectory -> ``G[B, N, n, n_e]`` (identity blocks around the
    4 x 3 attitude block ``L(q) H``; plain identity without a Lie-group state).  Host-side glue over ``states(prob)``."""
    X = states(prob)
    n, ne = prob.n, prob.ne
    G = np.zeros((prob.B, prob.N, n, ne))
    if ne == n:
        G[..., np.arange(n), np.arange(n)] = 1.0
        return G
    qs = 3
    for i in range(qs): G[..., i, i] = 1.0
    for i in range(qs + 4, n): G[..., i, i - 1] = 1.0
    w, x, y, z = (X[..., qs + i] for i in range(4))
    cols = ((-x, w, z, -y), (-y, -z, w, x), (-z, y, -x, w))          # columns of L(q) H (Rotations.jl grad-differential)
    for c, col in enumerate(cols):
        for r_, v in enumerate(col):
            G[..., qs + r_, qs + c] = v
    return G


def constraint_error_jacobians(prob, con):
    """``error_expansion!(jac, jac0, con, model, G, inds)`` (src/abstract_constraint.jl:282-303): the constraint Jacobians in the error
    state, ``[jac0_x G_k | jac0_u]`` -> ``[B, len(inds), p, n_e+m]``.  (The reference method only fills the state block of
    ``StateConstraint``s and the control block of ``ControlConstraint``s and leaves general stage constraints untouched; the full
    projection is what a solver needs and what the solver kernels use.)  Host-side glue over the device Jacobians."""
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    J0 = constraint_jacobians(prob, i)
    G = errstate_jacobian(prob)[:, first - 1:last]
    return np.concatenate([J0[..., :prob.n] @ G, J0[..., prob.n:]], axis=-1)


def multipliers(prob, con):
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    lam = np.empty((prob.B, last - first + 1, prob.constraints[i].p))
    prob._call("to_get_multipliers", i, K._dp(lam))
    return lam


def set_multipliers(prob, con, lam):
    i = _con_index(prob, con)
    first, last = prob.constraints.inds[i]
    lam = _bcast(lam, (prob.B, last - first + 1, prob.constraints[i].p), "lambda")
    prob._call("to_set_multipliers", i, K._dp(lam))


def penalty(prob, con):
    mu = C.c_double()
    prob._call("to_get_penalty", _con_index(prob, con), C.byref(mu))
    return mu.value


def set_penalty(prob, con, mu):
    prob._call("to_set_penalty", _con_index(prob, con), float(mu))


def backward_algebra(prob):
    """0 / 1: which of the two mathematically identical arithmetic forms the next backward pass uses (``to_backward_algebra``)"""
    v = C.c_int32()
    prob._call("to_backward_algebra", C.byref(v))
    return int(v.value)


def kernel_choice(prob):
    """which kernels the next solver calls launch, as the library picks them from the problem's shape (``to_kernel_choice``) -> dict:
    ``linesearch`` ("generic" / "fast" / "compact"), ``backward`` ("thread", "warp_mma", "warp_dfma", "fragment", "dense_mma",
    "dense_dfma"), the flags ``cost_cached``, ``fastal``, ``rec_fused``, ``late_list``, ``inst_forward``, ``inst_backward`` and ``resident``
    (k_riccati_frag instances resident at once on the device, 0 off the record path)"""
    v = (C.c_int32 * len(K.CHOICE_FIELDS))()
    prob._call("to_kernel_choice", v)
    d = dict(zip(K.CHOICE_FIELDS, (int(x) for x in v)))
    d["linesearch"] = K.LINESEARCH_LOOPS[d["linesearch"]]
    d["backward"] = K.BACKWARD_KERNELS[d["backward"]]
    for f in ("cost_cached", "fastal", "rec_fused", "late_list", "inst_forward", "inst_backward"):
        d[f] = bool(d[f])
    return d


def solver_state(prob):
    B = prob.B
    rho, dV, alpha = np.empty(B), np.empty((B, 2)), np.empty(B)
    ls, bp = np.empty(B, dtype=np.int32), np.empty(B, dtype=np.int32)
    prob._call("to_get_solver_state", K._dp(rho), K._dp(dV), K._dp(alpha), K._ip(ls), K._ip(bp))
    return dict(rho=rho, dV=dV, alpha=alpha, ls_iters=ls, bp_status=bp)


def set_options(prob, **kw):
    """update the given solver options; options set by earlier calls are kept (the C entry point takes the complete struct)"""
    o = getattr(prob, "_options", None)
    if o is None:
        o = K.to_options()
        prob._default_options(o)
    for k, v in kw.items():
        if not hasattr(o, k):
            raise ArgumentError(f"unknown solver option {k}")
        setattr(o, k, v)
    prob._options = o
    prob._call("to_set_options", C.byref(o))


# ---- solve!(prob): Altro's AL-iLQR solve to convergence, per instance (C ABI to_solve; semantics in include/trajopt_b200.h, DESIGN.md 5d) ----
SOLVE_STATUS_NAMES = {K.SOLVE_UNSOLVED: "UNSOLVED", K.SOLVE_SUCCEEDED: "SOLVE_SUCCEEDED", K.SOLVE_MAX_ITERATIONS: "MAX_ITERATIONS",
                      K.SOLVE_MAX_ITERATIONS_OUTER: "MAX_ITERATIONS_OUTER", K.SOLVE_MAX_REGULARIZATION: "MAX_REGULARIZATION"}


class SolveStats:
    """per-instance results of ``solve``, arrays of length B: ``status`` (to_solve_status codes, names in SOLVE_STATUS_NAMES),
    ``iterations`` (all inner loops together), ``iterations_outer``, ``cost`` (the objective of the final trajectory), ``dJ`` and ``gradient``
    of the last iteration, ``c_max`` (max violation when the last inner loop ended).  The trajectories, multipliers and gains stay in the
    problem: ``states(prob)``, ``controls(prob)``, ``multipliers(prob, con)``, ``gains(prob)``."""

    FIELDS = ("status", "iterations", "iterations_outer", "cost", "dJ", "gradient", "c_max")

    def __init__(self, B):
        self.status = np.zeros(B, dtype=np.int32)
        self.iterations = np.zeros(B, dtype=np.int32)
        self.iterations_outer = np.zeros(B, dtype=np.int32)
        self.cost, self.dJ, self.gradient, self.c_max = np.zeros(B), np.zeros(B), np.zeros(B), np.zeros(B)

    def status_names(self):
        return [SOLVE_STATUS_NAMES.get(int(s), str(int(s))) for s in self.status]

    def __repr__(self):
        names, counts = np.unique(self.status_names(), return_counts=True)
        return (f"SolveStats(B={len(self.status)}, status={dict(zip(names.tolist(), counts.tolist()))}, "
                f"iterations {int(self.iterations.min())}..{int(self.iterations.max())})")


def solve_options(**options):
    """a ``to_solve_options`` with Altro's defaults (``to_default_solve_options``) and the given overrides; ArgumentError on unknown names"""
    o = K.to_solve_options()
    K.load_library().to_default_solve_options(C.byref(o))
    for k, v in options.items():
        if k not in dict(K.to_solve_options._fields_):
            raise ArgumentError(f"unknown solve option {k}")
        setattr(o, k, v)
    return o


def solve(prob, **options):
    """solve!(prob): Altro's AL-iLQR solve of every instance to its own stopping point (Altro 0.3 SolverOptions names: cost_tolerance,
    cost_tolerance_intermediate, gradient_tolerance, gradient_tolerance_intermediate, constraint_tolerance, iterations, iterations_inner,
    iterations_outer, dJ_counter_limit).  The AL schedule (penalty_initial, penalty_scaling, ...) and the regularisation options are the
    solver options of ``set_options``.  Returns a ``SolveStats``."""
    o = solve_options(**options)
    st = SolveStats(prob.B)
    prob._call("to_solve", C.byref(o), K._ip(st.status), K._ip(st.iterations), K._ip(st.iterations_outer), K._dp(st.cost), K._dp(st.dJ),
               K._dp(st.gradient), K._dp(st.c_max))
    return st
