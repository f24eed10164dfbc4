"""ctypes binding of the C ABI declared in ``include/trajopt_b200.h``.

The library (``libtrajopt_b200.so``, built in-tree from ``csrc/`` by ``__graft_entry__.build()``) is the
product: hand-written sm_90a kernels behind a plain-C boundary.  There is no Python/CPU fallback -- if the
library is missing, or no CUDA device is present when a problem is created, this module raises.

The ``Spec`` helpers build the ``to_spec`` description of a problem (the data the reference keeps in its
``Problem`` / ``Objective`` / ``ConstraintList`` structs, reference src/problem.jl:36-73).  They are plain data
and are reused by the tests to feed the CPU oracle the identical description.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# LIBTRAJOPT_B200 overrides the in-tree path (INTEGRATION.md; profiles/build_variants.sh uses it for A/B kernel builds)
LIB_PATH = os.environ.get("LIBTRAJOPT_B200") or os.path.join(_HERE, "libtrajopt_b200.so")

# error codes (include/trajopt_b200.h)
TO_OK, TO_EINVAL, TO_EDIM, TO_ECUDA, TO_ENOMEM, TO_ESTATE, TO_ECONE = 0, -1, -2, -3, -4, -5, -6

MODEL_DOUBLE_INTEGRATOR, MODEL_CARTPOLE, MODEL_QUADROTOR, MODEL_ACROBOT, MODEL_EXPR = 0, 1, 2, 3, 4
COST_DIAGONAL, COST_QUADRATIC, COST_DIAGONAL_QUAT, COST_EXPR = 0, 1, 2, 3
(OP_CONST, OP_X, OP_U, OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_NEG, OP_SIN, OP_COS, OP_EXP, OP_LOG, OP_SQRT, OP_POWC, OP_TANH,
 OP_ADDC, OP_MULC, OP_DIVC, OP_RDIVC, OP_RSUBC) = range(20)
EXPR_MAXLEN, EXPR_MAXCONST = 128, 64
CONE_ZERO, CONE_NEGATIVE_ORTHANT, CONE_SECOND_ORDER, CONE_IDENTITY, CONE_POSITIVE_ORTHANT = 0, 1, 2, 3, 4
CON_GOAL, CON_BOUND, CON_LINEAR, CON_CIRCLE, CON_SPHERE, CON_NORM, CON_COLLISION, CON_QUATVEC, CON_EXPR = 0, 1, 2, 3, 4, 5, 6, 7, 8
# to_solve_status
SOLVE_UNSOLVED, SOLVE_SUCCEEDED, SOLVE_MAX_ITERATIONS, SOLVE_MAX_ITERATIONS_OUTER, SOLVE_MAX_REGULARIZATION = 0, 1, 2, 3, 4
PHASE_EXPAND, PHASE_BACKWARD, PHASE_FORWARD, PHASE_LADDER, PHASE_ACCEPT, PHASE_COSTEXP, PHASE_LATE, PHASE_COUNT = 0, 1, 2, 3, 4, 5, 6, 8
# to_kernel_choice: the entries of choice[] in order, and the names of the TO_LS_* / TO_BK_* values
CHOICE_FIELDS = ("linesearch", "cost_cached", "backward", "fastal", "rec_fused", "late_list", "inst_forward", "inst_backward", "resident")
LINESEARCH_LOOPS = ("generic", "fast", "compact")
BACKWARD_KERNELS = ("thread", "warp_mma", "warp_dfma", "fragment", "dense_mma", "dense_dfma")

c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)


class to_cost_spec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("terminal", C.c_int32), ("Q", c_double_p), ("R", c_double_p), ("H", c_double_p),
                ("q", c_double_p), ("r", c_double_p), ("c", C.c_double), ("w", C.c_double), ("q_ref", c_double_p), ("q_ind", c_int32_p),
                ("prog_len", C.c_int32), ("nconst", C.c_int32), ("prog", c_int32_p), ("consts", c_double_p)]


class to_constraint_spec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("first", C.c_int32), ("last", C.c_int32), ("sense", C.c_int32), ("p", C.c_int32),
                ("flag", C.c_int32), ("ninds", C.c_int32), ("inds", c_int32_p), ("a", c_double_p), ("b", c_double_p),
                ("c", c_double_p), ("rad", c_double_p), ("val", C.c_double)]


class to_dynamics_spec(C.Structure):
    _fields_ = [("n_in", C.c_int32), ("m_in", C.c_int32), ("n_out", C.c_int32), ("discrete", C.c_int32), ("prog_len", C.c_int32), ("nconst", C.c_int32),
                ("prog", c_int32_p), ("consts", c_double_p)]


class to_spec(C.Structure):
    _fields_ = [("model", C.c_int32), ("n", C.c_int32), ("m", C.c_int32), ("N", C.c_int32), ("B", C.c_int32),
                ("device", C.c_int32), ("nparams", C.c_int32), ("params", c_double_p), ("dt", c_double_p), ("t0", C.c_double),
                ("ncost", C.c_int32), ("costs", C.POINTER(to_cost_spec)), ("cost_index", c_int32_p),
                ("ncon", C.c_int32), ("cons", C.POINTER(to_constraint_spec)), ("error_state", C.c_int32),
                ("ndyn", C.c_int32), ("dyn", C.POINTER(to_dynamics_spec)), ("dyn_index", c_int32_p), ("nx", c_int32_p), ("nu", c_int32_p)]


class to_options(C.Structure):
    _fields_ = [("bp_reg_increase_factor", C.c_double), ("bp_reg_max", C.c_double), ("bp_reg_min", C.c_double),
                ("bp_reg_initial", C.c_double), ("bp_reg_fp", C.c_double),
                ("line_search_lower_bound", C.c_double), ("line_search_upper_bound", C.c_double),
                ("iterations_linesearch", C.c_int32), ("backward_kernel", C.c_int32),
                ("max_state_value", C.c_double), ("max_control_value", C.c_double),
                ("penalty_initial", C.c_double), ("penalty_scaling", C.c_double), ("penalty_max", C.c_double), ("dual_max", C.c_double)]


class to_solve_options(C.Structure):
    _fields_ = [("cost_tolerance", C.c_double), ("cost_tolerance_intermediate", C.c_double), ("gradient_tolerance", C.c_double),
                ("gradient_tolerance_intermediate", C.c_double), ("constraint_tolerance", C.c_double),
                ("iterations", C.c_int32), ("iterations_inner", C.c_int32), ("iterations_outer", C.c_int32), ("dJ_counter_limit", C.c_int32)]


class to_queue_spec(C.Structure):
    _fields_ = [("M", C.c_int32), ("U0_shared", C.c_int32), ("x0", c_double_p), ("U0", c_double_p), ("xf", c_double_p),
                ("goal_objective", C.c_int32), ("goal_constraint", C.c_int32), ("params", c_double_p), ("nparams", C.c_int32), ("pad", C.c_int32)]


class to_queue_table(C.Structure):
    _fields_ = [("kind", C.c_int32), ("index", C.c_int32), ("len", C.c_int32), ("pad", C.c_int32), ("rows", c_double_p), ("rows2", c_double_p)]


QT_TIME_STEPS, QT_COST_WEIGHTS, QT_CONSTRAINT_DATA, QT_PENALTIES, QT_REFERENCE = 0, 1, 2, 3, 4


class to_mpc_spec(C.Structure):
    _fields_ = [("nsteps", C.c_int32), ("nparams", C.c_int32), ("plant_params", c_double_p), ("W", c_double_p), ("Xref", c_double_p),
                ("Uref", c_double_p), ("nref", C.c_int32), ("start", C.c_int32)]


def _dp(a):
    return None if a is None else a.ctypes.data_as(c_double_p)


def _ip(a):
    return None if a is None else a.ctypes.data_as(c_int32_p)


def _f64(a):
    return None if a is None else np.ascontiguousarray(np.asarray(a, dtype=np.float64))


class Spec:
    """Owns the numpy buffers behind a ``to_spec`` so the pointers stay valid."""

    def __init__(self, model, n, m, N, B, dt, costs, cost_index, cons, params=None, t0=0.0, device=0, error_state=False,
                 dyn=None, dyn_index=None, nx=None, nu=None):
        self.keep = []
        self.model, self.n, self.m, self.N, self.B = int(model), int(n), int(m), int(N), int(B)
        dt = _f64(dt)
        self.keep.append(dt)
        cs = (to_cost_spec * len(costs))()
        for i, c in enumerate(costs):
            if c["kind"] == COST_EXPR:
                prog = np.ascontiguousarray(np.asarray(c["prog"], dtype=np.int32).reshape(-1, 3))
                consts = _f64(c["consts"])
                self.keep += [prog, consts]
                cs[i] = to_cost_spec(COST_EXPR, int(c.get("terminal", False)), None, None, None, None, None, 0.0, 0.0, None, None,
                                     len(prog), len(consts), _ip(prog), _dp(consts) if len(consts) else None)
                continue
            Q, R, H, q, r = _f64(c["Q"]), _f64(c["R"]), _f64(c.get("H")), _f64(c["q"]), _f64(c["r"])
            if c["kind"] == COST_QUADRATIC:   # column-major for the ABI
                Q = np.ascontiguousarray(Q.T); R = np.ascontiguousarray(R.T)
                H = None if H is None else np.ascontiguousarray(H.T)
            q_ref = _f64(c.get("q_ref"))
            q_ind = None if c.get("q_ind") is None else np.ascontiguousarray(np.asarray(c["q_ind"], dtype=np.int32))
            self.keep += [Q, R, H, q, r, q_ref, q_ind]
            cs[i] = to_cost_spec(c["kind"], int(c.get("terminal", False)), _dp(Q), _dp(R), _dp(H), _dp(q), _dp(r), float(c.get("c", 0.0)),
                                 float(c.get("w", 0.0)), _dp(q_ref), _ip(q_ind), 0, 0, None, None)
        ci = np.ascontiguousarray(np.asarray(cost_index, dtype=np.int32))
        self.keep.append(ci)
        ks = (to_constraint_spec * max(1, len(cons)))()
        for i, k in enumerate(cons):
            inds = None if k.get("inds") is None else np.ascontiguousarray(np.asarray(k["inds"], dtype=np.int32))
            a, b, c3, rad = _f64(k.get("a")), _f64(k.get("b")), _f64(k.get("c")), _f64(k.get("rad"))
            if k["kind"] == CON_LINEAR:
                a = np.ascontiguousarray(a.T)   # column-major A
            self.keep += [inds, a, b, c3, rad]
            ks[i] = to_constraint_spec(k["kind"], int(k["first"]), int(k["last"]), int(k.get("sense", 0)), int(k.get("p", 0)),
                                       int(k.get("flag", 0)), 0 if inds is None else len(inds), _ip(inds), _dp(a), _dp(b), _dp(c3), _dp(rad),
                                       float(k.get("val", 0.0)))
        p = _f64(params)
        self.keep += [cs, ks, p]
        ds, di, nxv, nuv = None, None, None, None
        if dyn:     # hybrid problem: recorded programs, one model per knot (to_dynamics_spec)
            ds = (to_dynamics_spec * len(dyn))()
            for i, d in enumerate(dyn):
                prog = np.ascontiguousarray(np.asarray(d["prog"], dtype=np.int32).reshape(-1, 3))
                consts = _f64(d["consts"])
                self.keep += [prog, consts]
                ds[i] = to_dynamics_spec(int(d["n_in"]), int(d["m_in"]), int(d["n_out"]), int(bool(d.get("discrete", False))), len(prog), len(consts),
                                         _ip(prog), _dp(consts) if len(consts) else None)
            di = np.ascontiguousarray(np.asarray(dyn_index, dtype=np.int32))
            nxv = np.ascontiguousarray(np.asarray(nx, dtype=np.int32)); nuv = np.ascontiguousarray(np.asarray(nu, dtype=np.int32))
            self.keep += [ds, di, nxv, nuv]
        self.c = to_spec(self.model, self.n, self.m, self.N, self.B, int(device), 0 if p is None else len(p), _dp(p), _dp(dt), float(t0),
                         len(costs), cs, _ip(ci), len(cons), ks, int(bool(error_state)),
                         0 if not dyn else len(dyn), ds, _ip(di), _ip(nxv), _ip(nuv))
        self.dyn, self.dyn_index, self.nx, self.nu = dyn, dyn_index, nx, nu
        self.error_state = bool(error_state)
        self.costs, self.cost_index, self.cons, self.dt = costs, list(cost_index), cons, dt
        self.t0, self.device = float(t0), int(device)


_lib = None


def load_library():
    """dlopen the in-tree C-ABI library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    H = C.c_void_p
    sig = {
        "to_create": [C.POINTER(to_spec), C.POINTER(H)],
        "to_recorded_dims": [C.c_int32, C.c_int32, c_int32_p, c_int32_p],
        "to_destroy": [H], "to_default_options": [C.POINTER(to_options)], "to_set_options": [H, C.POINTER(to_options)],
        "to_set_stream": [H, C.c_void_p], "to_synchronize": [H],
        "to_dims": [H, c_int32_p, c_int32_p, c_int32_p, c_int32_p], "to_num_constraints": [H, c_int32_p],
        "to_constraint_info": [H, C.c_int32, c_int32_p, c_int32_p, c_int32_p, c_int32_p],
        "to_bounds": [H, C.c_int32, c_double_p, c_double_p],
        "to_set_initial_state": [H, c_double_p], "to_set_controls": [H, c_double_p], "to_set_states": [H, c_double_p],
        "to_set_goal_state": [H, c_double_p, C.c_int, C.c_int], "to_set_initial_time": [H, C.c_double, c_double_p],
        "to_get_states": [H, c_double_p], "to_get_controls": [H, c_double_p], "to_get_times": [H, c_double_p],
        "to_update_trajectory": [H, c_double_p, c_double_p, C.c_int32, C.c_int32], "to_shift_trajectory": [H, C.c_int32],
        "to_set_goal_states": [H, c_double_p, C.c_int, C.c_int], "to_update_trajectories": [H, c_double_p, c_double_p, C.c_int32, C.c_int32],
        "to_get_cost_terms": [H, c_double_p, c_double_p], "to_set_cost_terms": [H, c_double_p, c_double_p],
        "to_get_goal_values": [H, C.c_int32, c_double_p], "to_set_goal_values": [H, C.c_int32, c_double_p],
        "to_set_model_params": [H, c_double_p, C.c_int32], "to_get_model_params": [H, c_double_p],
        "to_set_time_steps": [H, c_double_p, c_double_p], "to_get_time_steps": [H, c_double_p, c_double_p],
        "to_set_integration": [H, C.c_int32], "to_get_integration": [H, c_int32_p],
        "to_constraint_data_len": [H, C.c_int32, C.POINTER(C.c_int32)], "to_set_constraint_data": [H, C.c_int32, c_double_p],
        "to_get_constraint_data": [H, C.c_int32, c_double_p],
        "to_cost_weights_len": [H, C.c_int32, C.POINTER(C.c_int32)], "to_set_cost_weights": [H, C.c_int32, c_double_p],
        "to_get_cost_weights": [H, C.c_int32, c_double_p],
        "to_rollout": [H], "to_expand": [H], "to_get_dynamics_jacobians": [H, c_double_p],
        "to_cost": [H, c_double_p], "to_cost_knots": [H, c_double_p], "to_cost_gradient": [H, c_double_p], "to_cost_hessian": [H, c_double_p],
        "to_eval_constraints": [H, C.c_int32, c_double_p], "to_constraint_jacobians": [H, C.c_int32, c_double_p],
        "to_constraint_hessians": [H, C.c_int32, c_double_p, c_double_p],
        "to_max_violation": [H, c_double_p], "to_merit": [H, c_double_p], "to_al_expansion": [H, c_double_p, c_double_p],
        "to_projection": [H, C.c_int32, C.c_int32, C.c_int32, c_double_p, c_double_p],
        "to_grad_projection": [H, C.c_int32, C.c_int32, C.c_int32, c_double_p, c_double_p],
        "to_hess_projection": [H, C.c_int32, C.c_int32, C.c_int32, c_double_p, c_double_p, c_double_p],
        "to_backward": [H, c_int32_p], "to_forward": [H, c_double_p, c_double_p], "to_ilqr_step": [H, C.c_int32], "to_al_update": [H],
        "to_get_gains": [H, c_double_p, c_double_p], "to_get_multipliers": [H, C.c_int32, c_double_p],
        "to_set_multipliers": [H, C.c_int32, c_double_p], "to_get_penalty": [H, C.c_int32, c_double_p], "to_set_penalty": [H, C.c_int32, C.c_double],
        "to_set_penalties": [H, C.c_int32, c_double_p], "to_get_penalties": [H, C.c_int32, c_double_p],
        "to_get_solver_state": [H, c_double_p, c_double_p, c_double_p, c_int32_p, c_int32_p],
        "to_reduce_merit": [H], "to_reduce_merit_async": [H, C.c_void_p], "to_merit_device_ptr": [H, C.POINTER(C.c_void_p)],
        "to_set_phase_timing": [H, C.c_int], "to_get_phase_times": [H, c_double_p, C.POINTER(C.c_int64), C.c_int],
        "to_algorithmic_bytes": [H, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)],
        "to_backward_algebra": [H, c_int32_p], "to_kernel_choice": [H, c_int32_p], "to_error_state_dim": [H, c_int32_p], "to_state_diff": [H, c_double_p, c_double_p], "to_get_error_dynamics": [H, c_double_p],
        "to_error_expansion": [H, c_double_p, c_double_p], "to_get_expansion_records": [H, c_double_p],
        "to_default_solve_options": [C.POINTER(to_solve_options)],
        "to_solve": [H, C.POINTER(to_solve_options), c_int32_p, c_int32_p, c_int32_p, c_double_p, c_double_p, c_double_p, c_double_p],
        "to_mpc_setup": [H, C.POINTER(to_mpc_spec)], "to_mpc_run": [H, C.c_int32, C.c_int32], "to_mpc_history": [H, c_double_p, c_double_p, c_double_p],
        "to_mpc_solve": [H, C.c_int32, C.POINTER(to_solve_options)], "to_mpc_solve_history": [H, c_int32_p, c_int32_p, c_int32_p, c_double_p],
        "to_solve_queue": [H, C.POINTER(to_queue_spec), C.POINTER(to_solve_options), c_int32_p, c_int32_p, c_int32_p, c_double_p, c_double_p,
                           c_double_p, c_double_p, c_double_p, c_double_p],
        "to_solve_queue_tables": [H, C.POINTER(to_queue_spec), C.POINTER(to_queue_table), C.c_int32, C.POINTER(to_solve_options), c_int32_p,
                                  c_int32_p, c_int32_p, c_double_p, c_double_p, c_double_p, c_double_p, c_double_p, c_double_p],
    }
    for name, args in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    lib.to_last_error.argtypes = [H]
    lib.to_last_error.restype = C.c_char_p
    lib.to_launch_count.argtypes = [H]
    lib.to_launch_count.restype = C.c_int64
    _lib = lib
    return lib


EXPORTED_SYMBOLS = [
    "to_create", "to_recorded_dims", "to_destroy", "to_last_error", "to_default_options", "to_set_options", "to_set_stream", "to_synchronize", "to_dims",
    "to_num_constraints", "to_constraint_info", "to_bounds", "to_set_initial_state", "to_set_controls", "to_set_states",
    "to_set_goal_state", "to_set_initial_time", "to_get_states", "to_get_controls", "to_get_times", "to_rollout", "to_expand",
    "to_get_dynamics_jacobians", "to_cost", "to_cost_knots", "to_cost_gradient", "to_cost_hessian", "to_eval_constraints",
    "to_constraint_jacobians", "to_constraint_hessians", "to_max_violation", "to_merit", "to_al_expansion", "to_projection", "to_grad_projection",
    "to_hess_projection", "to_backward", "to_forward", "to_ilqr_step", "to_al_update", "to_get_gains", "to_get_multipliers",
    "to_set_multipliers", "to_get_penalty", "to_set_penalty", "to_set_penalties", "to_get_penalties", "to_get_solver_state", "to_reduce_merit", "to_reduce_merit_async", "to_merit_device_ptr", "to_update_trajectory", "to_shift_trajectory",
    "to_set_goal_states", "to_update_trajectories", "to_get_cost_terms", "to_set_cost_terms", "to_get_goal_values", "to_set_goal_values",
    "to_set_model_params", "to_get_model_params", "to_set_time_steps", "to_get_time_steps", "to_set_integration", "to_get_integration", "to_constraint_data_len", "to_set_constraint_data", "to_get_constraint_data",
    "to_cost_weights_len", "to_set_cost_weights", "to_get_cost_weights",
    "to_set_phase_timing", "to_get_phase_times", "to_launch_count", "to_algorithmic_bytes",
    "to_backward_algebra", "to_kernel_choice", "to_error_state_dim", "to_state_diff", "to_get_error_dynamics", "to_error_expansion",
    "to_get_expansion_records", "to_default_solve_options", "to_solve", "to_mpc_setup", "to_mpc_run", "to_mpc_history",
    "to_mpc_solve", "to_mpc_solve_history", "to_solve_queue", "to_solve_queue_tables",
]


class TrajOptError(RuntimeError):
    pass


def recorded_dims(nx_max, nu_max):
    """to_recorded_dims: the padded size class ``(n, m)`` -- (4, 2), (8, 4) or (16, 8) -- a recorded-program problem runs on when its largest
    per-knot state dimension is ``nx_max`` and its largest per-knot control dimension ``nu_max``.  Raises ``DimensionMismatch`` past (16, 8)."""
    lib = load_library()
    n, m = C.c_int32(), C.c_int32()
    rc = lib.to_recorded_dims(int(nx_max), int(nu_max), C.byref(n), C.byref(m))
    if rc == TO_EDIM:
        raise DimensionMismatch(f"recorded-program models: at most 16 states and 8 controls per knot, the largest has ({nx_max}, {nu_max})")
    if rc != TO_OK:
        raise ArgumentError(f"recorded-program models: no size class for ({nx_max}, {nu_max})")
    return n.value, m.value


class DimensionMismatch(TrajOptError):   # Julia DimensionMismatch (reference src/problem.jl:64-68)
    pass


class ArgumentError(TrajOptError, ValueError):   # Julia ArgumentError (reference src/problem.jl:87-91, src/constraints.jl:712)
    pass


def check(lib, handle, rc):
    if rc == TO_OK:
        return
    msg = lib.to_last_error(handle)
    msg = msg.decode() if msg else f"error {rc}"
    if rc == TO_EDIM:
        raise DimensionMismatch(msg)
    if rc == TO_EINVAL:
        raise ArgumentError(msg)
    raise TrajOptError(f"[{rc}] {msg}")
