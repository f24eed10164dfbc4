/* trajopt_b200.h -- C ABI of the H100-native batched problem-evaluation hot path of TrajectoryOptimization.jl.
 *
 * The reference (/root/reference, v0.7.1) is pure Julia and has no FFI: its "operator API" is the set of
 * Julia functions a solver (Altro.jl) calls on a `Problem`.  Each entry point below replaces one of those
 * calls for a BATCH of B independent problem instances that share model / objective / constraints and
 * differ in x0, X, U, multipliers -- and, after a per-instance goal call (to_set_goal_states,
 * to_update_trajectories, to_set_cost_terms), in the linear cost terms q, r and the Goal constraint values
 * (goal state / tracking reference per instance) -- and, after to_set_model_params, in the model parameters (mass,
 * inertia, lengths, motor constants, gravity) -- and, after to_set_constraint_data, in the constraint data (bounds, obstacles, collision
 * radii, norm values, linear right-hand sides) -- and, after to_set_cost_weights, in the cost weights Q, R, H, c, w -- and, after to_set_penalties, in the AL penalties -- and, after to_set_time_steps, in the time steps and initial time.  Every function cites the reference interface it stands in for.  The
 * Julia-side binding (ccall) that a maintainer adds is shown in INTEGRATION.md.
 *
 * Conventions
 *   - all functions return 0 on success or a negative TO_E* code; to_last_error() gives the message
 *     (the analogue of the reference's DimensionMismatch / ArgumentError exceptions, src/problem.jl:64-68,87-91).
 *     Nothing throws across the ABI.
 *   - host arrays are caller-owned, instance-major, Julia column-major within an instance:
 *       X[B][N][n]  == Julia Array{Float64,3}(n, N, B)        U[B][N-1][m] == Array(m, N-1, B)
 *       matrices are column-major (Julia), knot ranges and indices are 1-based like the reference.
 *   - device memory is owned by the library behind the opaque handle; one handle <-> one GPU <-> one stream;
 *     a handle is not thread-safe.  Multi-GPU = one process/handle per device, batch sharded (no data-path
 *     collective; the global merit all-reduce runs on to_merit_device_ptr()).
 *   - there is NO CPU fallback: every compute entry point launches sm_90a kernels or fails.
 */
#ifndef TRAJOPT_B200_H
#define TRAJOPT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TO_OK 0
#define TO_EINVAL (-1)   /* invalid argument (ArgumentError) */
#define TO_EDIM (-2)     /* dimension mismatch (DimensionMismatch, src/problem.jl:64-68, src/constraint_list.jl:108-110) */
#define TO_ECUDA (-3)    /* CUDA runtime failure */
#define TO_ENOMEM (-4)
#define TO_ESTATE (-5)   /* call order violated (e.g. backward pass before expansion) */
#define TO_ECONE (-6)    /* "Invalid second-order cone projection" (src/cones.jl:91,124) */

/* RobotZoo / example models on the path (SURVEY 8 a2) */
enum to_model_id {
    TO_MODEL_DOUBLE_INTEGRATOR = 0, /* examples/quickstart.jl:11-23 ; n = 2*dim, m = dim, params[0] = mass */
    TO_MODEL_CARTPOLE = 1,          /* docs/src/model.md:14-51 ; params = mc, mp, l, g */
    TO_MODEL_QUADROTOR = 2,         /* examples/Quadrotor.ipynb cells 4,8 ; params = mass, J1..3, g1..3, motor_dist, kf, km */
    TO_MODEL_ACROBOT = 3,           /* RobotZoo.Acrobot ; params = l1,l2,m1,m2,J1,J2,friction,g */
    TO_MODEL_EXPR = 4               /* user dynamics recorded as programs, one per knot allowed (hybrid / variable-dimension models, src/dynamics.jl:15-31,
                                       test/hybrid_dynamics_model.jl): to_spec.dyn, dyn_index, nx, nu.  Costs are given on the padded
                                       class layout, a knot's own entries first: TO_COST_DIAGONAL, TO_COST_QUADRATIC (dense Q, R, H) and
                                       TO_COST_EXPR (the Python Problem refuses TO_COST_DIAGONAL_QUAT
                                       on user models: quaternion costs are for the built-in rigid body).  Pad controls need a positive
                                       curvature of their own (unit R diagonal, or 0.5 u_j^2 in a program) so that Quu stays positive
                                       definite; they stay zero. */
};

/* The explicit rule that discretises the dynamics (RobotDynamics' Euler, RK2, RK3, RK4 with zero-order hold on u; `Problem(...; integration)`,
 * src/problem.jl:32, :119-123).  See to_set_integration. */
enum to_integration { TO_EULER = 1, TO_RK2 = 2, TO_RK3 = 3, TO_RK4 = 4 };

/* QuadraticCostFunction (src/cost_functions.jl:326-347 DiagonalCost, :417-454 QuadraticCost) */
/* DiagonalQuatCost / QuatLQRCost (src/lie_costs.jl:33-95, :129-139): a DiagonalCost plus w * min(1 + q_ref'p, 1 - q_ref'p), p = x[q_ind] */
/* Generic (user-defined) cost: the reference lets users subtype CostFunction and get gradient!/hessian! from ForwardDiff through
 * RD.@autodiff (docs/src/costfunction_interface.md:30-50, test/nlcosts.jl:4-19).  Here the user function arrives as a straight-line
 * PROGRAM (SSA, one value per instruction, the last one is the cost) recorded by the host API, and the kernels evaluate it with
 * second-order forward-mode dual numbers (SURVEY 8 f4).  Instruction i = {op, a, b}: operands are indices of earlier instructions,
 * of the state / control vector (TO_OP_X / TO_OP_U), or of the constant table (TO_OP_CONST; TO_OP_POWC: b).  At the terminal knot the
 * program is evaluated with u = 0 and only the state derivatives are taken (the reference's zero terminal control). */
enum to_cost_kind { TO_COST_DIAGONAL = 0, TO_COST_QUADRATIC = 1, TO_COST_DIAGONAL_QUAT = 2, TO_COST_EXPR = 3 };
enum to_expr_op { TO_OP_CONST = 0, TO_OP_X = 1, TO_OP_U = 2, TO_OP_ADD = 3, TO_OP_SUB = 4, TO_OP_MUL = 5, TO_OP_DIV = 6, TO_OP_NEG = 7,
                  TO_OP_SIN = 8, TO_OP_COS = 9, TO_OP_EXP = 10, TO_OP_LOG = 11, TO_OP_SQRT = 12, TO_OP_POWC = 13 /* a ^ const[b] */, TO_OP_TANH = 14,
                  /* one operand taken from the constant table: a (op) const[b] */
                  TO_OP_ADDC = 15, TO_OP_MULC = 16, TO_OP_DIVC = 17 /* a / c */, TO_OP_RDIVC = 18 /* c / a */, TO_OP_RSUBC = 19 /* c - a */ };
#define TO_EXPR_MAXLEN 128
#define TO_EXPR_MAXCONST 64
typedef struct {
    int32_t kind;     /* to_cost_kind */
    int32_t terminal; /* `terminal` flag of the cost (LQRObjective sets it on the last cost, src/objective.jl:154,180) */
    const double* Q;  /* DIAGONAL: n diagonal entries ; QUADRATIC: n*n column-major */
    const double* R;  /* DIAGONAL: m ; QUADRATIC: m*m column-major */
    const double* H;  /* QUADRATIC: m*n column-major cross term u'Hx, or NULL (zero) */
    const double* q;  /* n */
    const double* r;  /* m */
    double c;
    double w;               /* DIAGONAL_QUAT: weight of the geodesic term */
    const double* q_ref;    /* DIAGONAL_QUAT: reference quaternion (4, scalar first); else NULL */
    const int32_t* q_ind;   /* DIAGONAL_QUAT: 1-based state indices of the quaternion (4); NULL = 4:7 (src/lie_costs.jl:64) */
    int32_t prog_len;       /* EXPR: number of instructions (<= TO_EXPR_MAXLEN); Q, R, q, r may be NULL */
    int32_t nconst;         /* EXPR: number of constants (<= TO_EXPR_MAXCONST) */
    const int32_t* prog;    /* EXPR: prog_len x {op, a, b} */
    const double* consts;   /* EXPR */
} to_cost_spec;

/* One dynamics model of a hybrid problem: `RD.@autodiff struct M <: ContinuousDynamics` + `RD.dynamics(::M, x, u)` recorded as a program
 * (to_expr_op; inputs x[0..n_in), u[0..m_in); the LAST n_out instructions are the outputs), discretised with the problem's explicit rule (to_set_integration),
 * or -- `discrete` = 1 -- a jump map x+ = g(x, u) applied as is (n_out may differ from n_in: the state dimension changes there). */
typedef struct {
    int32_t n_in, m_in, n_out, discrete;
    int32_t prog_len, nconst;
    const int32_t* prog;
    const double* consts;
} to_dynamics_spec;

/* ConstraintSense (src/cones.jl:17-61) */
enum to_cone { TO_CONE_ZERO = 0 /* Equality */, TO_CONE_NEGATIVE_ORTHANT = 1 /* Inequality */, TO_CONE_SECOND_ORDER = 2,
               TO_CONE_IDENTITY = 3, TO_CONE_POSITIVE_ORTHANT = 4 };

/* AbstractConstraint subtypes (src/constraints.jl) */
enum to_con_kind {
    TO_CON_GOAL = 0,   /* GoalConstraint :22-87      a = xf[ninds], inds = 1-based state indices             */
    TO_CON_BOUND = 1,  /* BoundConstraint :644-783   a = z_max[n+m], b = z_min[n+m] (+-Inf = unbounded)        */
    TO_CON_LINEAR = 2, /* LinearConstraint :103-150  a = A[p x w] col-major, b = b[p], flag = 0 state | 1 control, sense */
    TO_CON_CIRCLE = 3, /* CircleConstraint :168-233  a = xc[p], b = yc[p], rad = r[p], inds = {xi, yi} (1-based) */
    TO_CON_SPHERE = 4, /* SphereConstraint :249-326  a,b,c = centers, rad, inds = {xi, yi, zi}                 */
    TO_CON_NORM = 5,   /* NormConstraint :438-521    val, inds = 1-based indices into z, sense (orthant | SOC)   */
    TO_CON_COLLISION = 6, /* CollisionConstraint :341-389  val = radius, inds = {x1[D], x2[D]} 1-based state indices (ninds = 2D): r^2 - |x[x1]-x[x2]|^2 <= 0.
                            StateBound / ControlBound :547-631 are TO_CON_BOUND with the other block unbounded. */
    TO_CON_EXPR = 8,     /* user constraint recorded as a program (RD.@autodiff struct ... <: StageConstraint, docs/src/constraint_interface.md:52-72):
                            inds = prog_len x {op, a, b} (ninds = 3 prog_len, to_expr_op as for TO_COST_EXPR), a = constants (flag = their number),
                            p = output dimension: the values of the LAST p instructions; sense; Jacobian by forward-mode AD on the device */
    TO_CON_QUATVEC = 7   /* QuatVecEq :938-965  a = qf (4, scalar first), inds = qind (4, 1-based; NULL = 4:7): with q = normalize(x[qind]) and
                            qf flipped when qf'q < 0, c = q[2:4] - qf[2:4]; Equality, p = 3 */
};
typedef struct {
    int32_t kind;        /* to_con_kind */
    int32_t first, last; /* knot range first:last, 1-based inclusive (add_constraint!, src/constraint_list.jl:103-134) */
    int32_t sense;       /* to_cone; ignored for GOAL (Equality) and BOUND/CIRCLE/SPHERE (Inequality) */
    int32_t p;           /* rows for LINEAR / number of obstacles for CIRCLE, SPHERE; ignored otherwise */
    int32_t flag;
    int32_t ninds;
    const int32_t* inds;
    const double* a;
    const double* b;
    const double* c;
    const double* rad;
    double val;
} to_constraint_spec;

/* Problem(model, obj, x0, tf; constraints, ...)  src/problem.jl:79-123 */
typedef struct {
    int32_t model;           /* to_model_id */
    int32_t n, m;            /* state / control dimension (checked against the model, src/problem.jl:64-68) */
    int32_t N;               /* knot points == length(obj) (src/problem.jl:95) */
    int32_t B;               /* batch: independent problem instances on this device */
    int32_t device;          /* CUDA device ordinal */
    int32_t nparams;
    const double* params;    /* model parameters, NULL = the model's defaults */
    const double* dt;        /* N-1 time steps (vector dt allowed, test/problems_tests.jl:79-82) */
    double t0;
    int32_t ncost;           /* distinct cost functions */
    const to_cost_spec* costs;
    const int32_t* cost_index; /* N entries, 0-based index into costs (Objective.cost, src/objective.jl:27-45) */
    int32_t ncon;
    const to_constraint_spec* cons; /* ConstraintList, in add_constraint! order */
    int32_t error_state;     /* 1: the solver kernels (backward / forward pass) work on the ERROR STATE of a Lie-group model, as Altro does when
                                RD.errstate_dim(model) != n: the Quadrotor's quaternion (x[4:7]) contributes 3 dimensions, n_e = 12.  State-difference
                                Jacobian G(x) = blkdiag(I3, L(q) H, I6) (Rotations.jl grad-differential), dynamics A_e = G_{k+1}' A G_k, B_e = G_{k+1}' B,
                                cost expansion G'lxx G + grad^2-differential, dx = state_diff(xbar, x) with the Cayley map.  The reference's hooks for
                                it: src/abstract_constraint.jl:282-303 (error_expansion! of constraint Jacobians), src/lie_costs.jl.  0: full state. */
    /* TO_MODEL_EXPR only (else 0 / NULL): `Problem(models::Vector{<:DiscreteDynamics}, ...)`, src/problem.jl:36-73 with RD.dims(models), src/dynamics.jl:15-31.
       n, m are the padded size class to_recorded_dims gives for the LARGEST per-knot state / control dimensions (any other n, m is refused
       with TO_EDIM); knot k has nx[k] <= n states and nu[k] <= m controls, stored in the first entries of the n- / m-sized slots (the rest stays zero: costs and constraints are described on the padded [x(n); u(m)] layout, with unit weights on the
       unused controls so that Quu stays positive definite).  Model dyn[dyn_index[k]] maps knot k to k+1: n_in = nx[k], m_in = nu[k], n_out = nx[k+1]
       (checked: the reference's DimensionMismatch "Model mismatch at time step k"). */
    int32_t ndyn;
    const to_dynamics_spec* dyn;
    const int32_t* dyn_index;   /* N-1 entries, 0-based */
    const int32_t* nx;          /* N entries */
    const int32_t* nu;          /* N entries (nu[N-1] = nu[N-2], as RD.dims does) */
} to_spec;

/* Solver options on the path (Altro.jl SolverOptions, restated in oracle/oracle.hpp `Options`) */
typedef struct {
    double bp_reg_increase_factor, bp_reg_max, bp_reg_min, bp_reg_initial, bp_reg_fp;
    double line_search_lower_bound, line_search_upper_bound;
    int32_t iterations_linesearch;
    int32_t backward_kernel;   /* 0 = automatic; 1 = warp-per-instance Riccati kernel; 2 = thread-per-instance kernel (n <= 4, m <= 2,
                                  Goal/Bound constraints only, else ignored); error-state problems: 3 = generic DFMA kernel on the full
                                  materialised expansion, 5 = shared-memory tensor kernel on the compact expansion (automatic = the
                                  register-resident fragment kernel when the problem is compact). Not a solver option of the reference:
                                  a tuning / test knob. */
    double max_state_value, max_control_value;
    double penalty_initial, penalty_scaling, penalty_max, dual_max;
} to_options;

typedef struct to_handle to_handle;

/* ---- lifecycle -------------------------------------------------------------------------------------- */
int to_create(const to_spec* spec, to_handle** out);                 /* Problem(...)           src/problem.jl:79-111 */
/* The padded size class (n, m) of a recorded-program problem (TO_MODEL_EXPR) whose largest per-knot state dimension is nx_max and largest
 * per-knot control dimension is nu_max: the smallest of (4, 2), (8, 4) and (16, 8) that holds both.  TO_EDIM past (16, 8); TO_EINVAL for
 * nx_max < 1, nu_max < 0 or a NULL output.  to_spec.n, m of such a problem must be this class. */
int to_recorded_dims(int32_t nx_max, int32_t nu_max, int32_t* n, int32_t* m);
int to_destroy(to_handle* h);
const char* to_last_error(const to_handle* h);                       /* h may be NULL: error of the last failed to_create */
int to_default_options(to_options* o);
int to_set_options(to_handle* h, const to_options* o);
int to_set_stream(to_handle* h, void* cuda_stream);                  /* run on the caller's stream (e.g. torch's current stream) */
int to_synchronize(to_handle* h);
int to_dims(const to_handle* h, int32_t* n, int32_t* m, int32_t* N, int32_t* B); /* RD.dims(prob)  src/problem.jl:139-147 */
int to_num_constraints(const to_handle* h, int32_t* p_per_knot /*[N]*/);         /* num_constraints(prob) src/problem.jl:206 */
int to_constraint_info(const to_handle* h, int32_t con, int32_t* p, int32_t* sense, int32_t* first, int32_t* last);
int to_bounds(const to_handle* h, int32_t con, double* lower /*[p]*/, double* upper /*[p]*/); /* lower_bound/upper_bound src/abstract_constraint.jl:97-123 */

/* ---- setters / getters (host arrays, instance-major) ------------------------------------------------ */
/* The setters enqueue their host-to-device copy on the handle's stream and return: the host buffer must stay valid (and unchanged) until the next
 * synchronising call on the handle -- to_synchronize or any getter.  Getters copy back and synchronise the handle's stream before returning. */
int to_set_initial_state(to_handle* h, const double* x0 /*[B][n]*/);          /* set_initial_state! src/problem.jl:270 */
int to_set_controls(to_handle* h, const double* U /*[B][N-1][m]*/);           /* initial_controls!  src/problem.jl:261 */
int to_set_states(to_handle* h, const double* X /*[B][N][n]*/);               /* initial_states!    src/problem.jl:253 */
int to_set_goal_state(to_handle* h, const double* xf /*[n]*/, int objective, int constraint); /* set_goal_state! src/problem.jl:294-310 */
int to_set_initial_time(to_handle* h, double t0, double* tf_out);             /* setinitialtime!    src/problem.jl:280 */
int to_get_states(to_handle* h, double* X /*[B][N][n]*/);                     /* states(prob)       src/problem.jl:175 */
int to_get_controls(to_handle* h, double* U /*[B][N-1][m]*/);                 /* controls(prob)     src/problem.jl:168 */
int to_get_times(to_handle* h, double* t /*[N]*/);                            /* gettimes(prob)     src/problem.jl:182 */

/* ---- MPC plumbing (SURVEY 8 f3; BASELINE config 5) ---------------------------------------------------------
 * update_trajectory!(obj, Z, start) src/objective.jl:207-212: knot i = 1..N of a tracking objective follows row
 * (start-1+i) of the reference: set_LQR_goal! (src/cost_functions.jl:245-254) q = -Q xf, r = -R uf, c untouched.
 * Xref [nref][n], Uref [nref][m] host arrays (start + N - 1 <= nref). Costs shared by several knots end up tracking
 * the last of them, exactly as the reference's aliased cost objects do. */
int to_update_trajectory(to_handle* h, const double* Xref, const double* Uref, int32_t nref, int32_t start);
/* Receding-horizon warm start, on the device: X_k <- X_{k+steps}, U_k <- U_{k+steps} (the tail repeats the last
 * control and state), multipliers move with their knots (the tail keeps its last value), x0 <- X_{1+steps},
 * t0 += the skipped dt. The caller then sets the measured state (to_set_initial_state) and re-rolls out. */
int to_shift_trajectory(to_handle* h, int32_t steps);

/* ---- per-instance goals / tracking references ---------------------------------------------------------------
 * The same operations per instance b.  Per instance the handle holds the linear terms q_b, r_b of every distinct cost (cost_index aliasing
 * kept: a cost shared by several knots tracks the last of them, per instance) and the values of every Goal constraint; the weights Q, R, H,
 * c and w are per instance after to_set_cost_weights (below); q_ref, program costs and every other constraint stay shared.  Until the first per-instance call there is no
 * per-instance data and every kernel runs as before.  The first per-instance call copies the shared values into every instance, then applies
 * its change; a later shared to_set_goal_state / to_update_trajectory writes through to every instance (the later call wins).
 * to_shift_trajectory leaves the objective alone: an MPC loop calls to_update_trajectories with the next start.  Multi-GPU: each rank passes
 * its shard's rows, as for x0.  The quaternion cost's w / q_ref and program costs keep their shared values (program costs have no linear
 * term); every solver path takes the per-instance values.  Not available (TO_EINVAL) on hybrid problems. */
int to_set_goal_states(to_handle* h, const double* xf /*[B][n]*/, int objective, int constraint);    /* set_goal_state! per instance */
int to_update_trajectories(to_handle* h, const double* Xref /*[B][nref][n]*/, const double* Uref /*[B][nref][m]*/,
                           int32_t nref, int32_t start);                                            /* update_trajectory! per instance (TO_EDIM: nref < start + N - 1) */
int to_get_cost_terms(to_handle* h, double* q /*[B][ncost][n]*/, double* r /*[B][ncost][m]*/);     /* the shared values broadcast when none are set */
int to_set_cost_terms(to_handle* h, const double* q, const double* r);                              /* set_LQR_goal!(obj[k], ...) per instance, raw terms */
int to_get_goal_values(to_handle* h, int32_t con, double* vals /*[B][p]*/);                        /* a Goal constraint's xf[inds] of every instance */
int to_set_goal_values(to_handle* h, int32_t con, const double* vals);                             /* ... set per instance (TO_EINVAL: not a Goal) */

/* ---- per-instance model parameters ---------------------------------------------------------------------------
 * Instance b integrates its dynamics with its own parameter vector (a Problem owns its model, src/problem.jl:36-73): the entries and order of
 * to_spec.params, nparams = 1 (DoubleIntegrator), 4 (Cartpole), 10 (Quadrotor), 8 (Acrobot).  Until the first call every instance uses the
 * shared to_spec.params and every kernel runs as before.  A batch whose instance b holds p_b computes, bit for bit, what instance b of a batch
 * created with p_b as to_spec.params computes.  X is not rolled out again: the next rollout / expansion / line search / solve uses the new
 * values.  TO_EDIM: nparams is not the model's count.  TO_EINVAL: a hybrid problem, a non-finite entry, or a non-positive mass, inertia or
 * length the dynamics divide by (DoubleIntegrator mass; Cartpole mc, mp, l; Quadrotor mass, J1..J3; Acrobot l1, l2, m1, m2); the message names
 * the instance and the entry, and the rows stay as they were.  Multi-GPU: each rank passes its shard's rows, as for x0. */
int to_set_model_params(to_handle* h, const double* params /*[B][nparams]*/, int32_t nparams);
int to_get_model_params(to_handle* h, double* params /*[B][nparams]*/);                             /* the shared values broadcast when none are set */

/* ---- per-instance time steps -----------------------------------------------------------------------------------
 * Instance b integrates knot k with its own step dt[b][k], and its clock starts at t0[b]: its knot times are t0_b, t0_b + dt_b[0], ...  This is
 * what Problem(model, obj, x0_b, tf_b; t0 = t0_b, dt = dt_b) holds (src/problem.jl:16-29, 79-111).  Until the first call there is no table and
 * every kernel runs as before; t0 = NULL keeps the clocks (the first call starts them at the shared t0).  A batch whose instance b holds
 * (t0_b, dt_b) computes, bit for bit, what instance b of a batch created with that grid computes, on every solver path.  X is not rolled out
 * again.  to_get_times keeps returning the shared grid (to_spec.t0 and dt), as to_bounds keeps the shared bounds.  to_set_initial_time sets
 * the shared clock and every instance's; to_shift_trajectory advances each instance's clock by its own skipped steps and leaves the rows as
 * they are.  TO_EINVAL: a hybrid problem, a step that is non-finite or <= 0, a non-finite t0; the message names the instance and the knot, and
 * the table and clocks stay as they were.  Multi-GPU: each rank passes its shard's rows, as for x0. */
int to_set_time_steps(to_handle* h, const double* dt /*[B][N-1]*/, const double* t0 /*[B] or NULL: keep the clocks*/);
int to_get_time_steps(to_handle* h, double* dt /*[B][N-1]*/, double* t0 /*[B] or NULL*/);            /* the shared values broadcast when none are set */

/* ---- per-instance constraint data ----------------------------------------------------------------------------
 * Instance b evaluates constraint con with its own data (a Problem owns its ConstraintList, src/problem.jl:36-73).  One instance's row, len doubles:
 *   BOUND     2(n+m)  z_max[n+m] | z_min[n+m], +-Inf where the shared bound is +-Inf
 *   LINEAR    p       b[p]  (A stays shared)
 *   CIRCLE    3p      xc[p] | yc[p] | r[p]
 *   SPHERE    4p      xc[p] | yc[p] | zc[p] | r[p]
 *   NORM      1       val
 *   COLLISION 1       radius
 * to_constraint_data_len gives len (0 for GOAL, which has to_set_goal_values, and for QUATVEC / EXPR, whose constants stay shared).  Until the
 * first to_set_constraint_data there is no table and every kernel runs as before; the first call fills every instance with the shared data of
 * every constraint, then applies its rows.  The shape stays fixed: rows, knot ranges and the multiplier layout never change, so a BOUND row must
 * be finite exactly where the shared bound is, with the same infinities.  TO_EINVAL, with the instance and the entry named, and nothing changed:
 * a changed +-Inf pattern, z_max < z_min (src/constraints.jl:712), a non-finite entry of another kind, a NORM val < 0 (:451), a GOAL, QUATVEC or
 * EXPR constraint, a hybrid problem.  to_shift_trajectory leaves the data alone (obstacles live in the world frame); to_bounds keeps returning
 * the shared values.  A batch whose instance b holds d_b computes, bit for bit, what instance b of a batch created with d_b as the shared data
 * computes, on every solver path.  Multi-GPU: each rank passes its shard's rows, as for x0. */
int to_constraint_data_len(const to_handle* h, int32_t con, int32_t* len);                         /* doubles per instance of constraint con */
int to_set_constraint_data(to_handle* h, int32_t con, const double* data /*[B][len]*/);
int to_get_constraint_data(to_handle* h, int32_t con, double* data /*[B][len]*/);                  /* the shared values broadcast when none are set */

/* ---- per-instance cost weights -------------------------------------------------------------------------------
 * Instance b evaluates distinct cost `cost` (0-based index into to_spec.costs) with its own weights (a Problem owns its Objective,
 * src/problem.jl:36-73).  One instance's row, len doubles, in to_cost_spec order, matrices column-major:
 *   DIAGONAL       n+m+1          Qd[n] | Rd[m] | c
 *   QUADRATIC      n^2+m^2+mn+1   Q[n*n] | R[m*m] | H[m*n] | c
 *   DIAGONAL_QUAT  n+m+2          Qd[n] | Rd[m] | c | w
 *   EXPR           0              (the program's constants stay shared)
 * With the diagonal layouts entry i of z reads row[i], as in a row of the linear terms (q[n] | r[m]).  to_cost_weights_len gives len.  Until
 * the first to_set_cost_weights there is no table and every kernel runs as before; the first call fills every instance with the shared weights
 * of every cost, then applies its rows.  The shape stays fixed: the kind, terminal flag, q_ind and q_ref stay shared, and a QUADRATIC cost
 * whose shared H is zero keeps H zero in every row (the zero pattern selects kernel code).  Weights to_create would accept in a spec of that
 * kind are accepted (indefinite Q or R included, as the reference only warns).  TO_EINVAL, with the instance and the entry named, and nothing
 * changed: a non-finite entry, a non-zero H where the shared H is zero, an EXPR cost, a hybrid problem, a cost index out of range.  The linear
 * terms stay as they are (mutating cost.Q leaves cost.q alone); from then on to_set_goal_state(s) and to_update_trajectory(ies) set
 * q_b = -Q_b xf and r_b = -R_b uf with each instance's own weights, the shared setters writing through to every instance.  A batch whose
 * instance b holds w_b computes, bit for bit, what instance b of a batch created with w_b as the shared cost computes, on every solver path.
 * Multi-GPU: each rank passes its shard's rows, as for x0. */
int to_cost_weights_len(const to_handle* h, int32_t cost, int32_t* len);                            /* doubles per instance of distinct cost `cost` */
int to_set_cost_weights(to_handle* h, int32_t cost, const double* w /*[B][len]*/);
int to_get_cost_weights(to_handle* h, int32_t cost, double* w /*[B][len]*/);                       /* the shared values broadcast when none are set */

/* ---- integrator ------------------------------------------------------------------------------------------------
 * The explicit rule every kernel that steps the dynamics uses (rollout, dynamics expansion, line search): TO_EULER x+ = x + h f(x,u);
 * TO_RK2 (explicit midpoint); TO_RK3 (Kutta); TO_RK4, the default until the first call.  Each k_i is scaled by h before it is used, as
 * RobotDynamics does.  One rule holds for the whole batch; in a hybrid problem it applies to every continuous model and a discrete jump map
 * is still applied as it is.  The Jacobians, expansions and gains computed before the call are stale afterwards, as after to_set_time_steps;
 * X is not rolled out again.  TO_EINVAL, naming the code, with nothing changed: any other code (the implicit rules, ImplicitMidpoint and
 * HermiteSimpson, included: iLQR's rollout needs an explicit step). */
int to_set_integration(to_handle* h, int32_t rule);
int to_get_integration(const to_handle* h, int32_t* rule);

/* ---- closed-loop MPC on the device -------------------------------------------------------------------------------
 * A receding-horizon simulation of every instance without a host round trip per step.  MPC step j (j counts from the last setup) runs, bit
 * for bit, what this host-scripted loop of entry points computes:
 *   1. with a reference: to_update_trajectories(Xref, Uref, nref, start + j);
 *   2. to_rollout;  3. to_ilqr_step(iterations);
 *   4. record u_j = U[b][0] (to_get_controls) and the plan's merit J_j (to_merit);
 *   5. the plant: xp <- step(xp, u_j) (+) w_j, recorded as Xcl[j+1];
 *   6. to_shift_trajectory(1), then to_set_initial_state(xp).
 * The plant is the problem's model stepped once with the problem's integration rule over the instance's knot-0 time step (its own row after
 * to_set_time_steps), with the plant's parameter rows when the setup gave them, else the planner's (per instance when set).  (+) is the
 * inverse of to_state_diff: addition for vector-space states, the Cayley-map composition q (x) (1, phi) / sqrt(1 + phi'phi) on the
 * error-state Quadrotor's quaternion; w_j has n_e entries.  A run starts from xp = x0, so runs of T1 and T2 steps leave what one run of
 * T1 + T2 leaves.  Multipliers and penalties are shifted by step 6 and not otherwise updated; to_al_update or any setter may run between runs.
 * Not on hybrid problems; a problem whose every knot steps one continuous recorded model is a plant like any other, without a reference window
 * or plant parameters (it has no per-instance goals or parameters).
 * to_mpc_solve replaces steps 2-3 by a solve: step j runs, bit for bit,
 *   2. to_solve(o) (roll out from x0, merit, inner loops and outer steps; multipliers and penalties kept, as to_solve keeps them);
 *   3. record J_j = to_merit after the solve, and the step's status, iterations, iterations_outer and c_max as to_solve returns them;
 * with steps 1 and 4-6 as above.  Each step runs exactly o->iterations iterations with the stopping-rule checks and reads nothing back: every
 * instance is done within that budget, and the iterations after an instance stops leave it as it is (to_solve's own last iteration, in which
 * no instance is ACTIVE, is one of them).  The device takes each outer step only when every instance holds its own penalties: on a
 * constrained problem without a per-instance penalty table the first to_mpc_solve creates it, every row holding the shared penalties, as the
 * first to_set_penalties does (synchronous, once; bit for bit the shared penalties' results).  So the scripted equivalent is
 * to_set_penalties(con, shared mu) for every constraint, then the loop.  to_mpc_run and to_mpc_solve steps may alternate within one setup. */
typedef struct {
    int32_t nsteps;              /* the steps the setup holds room for (>= 1) */
    int32_t nparams;             /* entries of a plant row, as to_set_model_params takes them */
    const double* plant_params;  /* [B][nparams] or NULL: the planner's parameters */
    const double* W;             /* [B][nsteps][n_e] disturbances or NULL: none */
    const double* Xref;          /* [B][nref][n] or NULL: no reference window */
    const double* Uref;          /* [B][nref][m] (with Xref) */
    int32_t nref, start;         /* step j tracks rows start - 1 + j .. start - 2 + j + N (1-based start) */
} to_mpc_spec;
/* Synchronous: checks the inputs and copies them to device buffers of the handle, allocates the history and resets the step counter; with a
 * reference it creates the per-instance linear terms as to_update_trajectories does.  TO_EDIM: start - 1 + (nsteps - 1) + N > nref, or a
 * plant row of the wrong length.  TO_EINVAL, naming the instance: a non-finite entry, a plant row to_set_model_params would refuse; nsteps
 * < 1, a hybrid problem.  A refused setup leaves the previous one as it was. */
int to_mpc_setup(to_handle* h, const to_mpc_spec* spec);
/* Asynchronous, like to_ilqr_step: enqueues `steps` MPC steps of `iterations` iLQR iterations each on the handle's stream(s) and returns.
 * TO_ESTATE before any setup; TO_EDIM when the steps done since the setup + steps > nsteps; TO_EINVAL when steps or iterations < 1; the
 * checks of to_ilqr_step.  The host clocks advance as to_shift_trajectory(1) advances them; to_get_cost_terms reads the rows the last window
 * wrote. */
int to_mpc_run(to_handle* h, int32_t steps, int32_t iterations);
/* The history of the s steps run since the setup, and synchronises: Xcl [B][s+1][n] (row j: the state step j started from; row s: where the
 * last step ended, x0 when s = 0), Ucl [B][s][m], J [B][s].  Any output may be NULL.  TO_ESTATE before any setup. */
int to_mpc_history(to_handle* h, double* Xcl, double* Ucl, double* J);
struct to_solve_options;   /* (declared with to_solve below) */
/* Asynchronous, like to_mpc_run: enqueues `steps` MPC steps whose plan is to_solve(o) (above) and returns.  TO_ESTATE before any setup;
 * TO_EDIM when the steps done since the setup + steps > nsteps; TO_EINVAL when steps < 1, for the options to_solve refuses (with its
 * messages), and for a constrained problem of a recorded-program model (it has no per-instance penalties); the checks of to_solve.  Every
 * check comes before anything is enqueued or changed. */
int to_mpc_solve(to_handle* h, int32_t steps, const struct to_solve_options* o);
/* The solve statistics of the s steps run since the setup, and synchronises: status, iterations, iterations_outer, c_max [B][s] each, as
 * to_solve returns them.  A step to_mpc_run took holds status -1, iterations 0, iterations_outer 0, c_max NaN.  Any output may be NULL.
 * TO_ESTATE before any setup. */
int to_mpc_solve_history(to_handle* h, int32_t* status, int32_t* iterations, int32_t* iterations_outer, double* c_max);

/* ---- kernel 1: batched rollout (+ dual-number Jacobians) ------------------------------------------------- */
int to_rollout(to_handle* h);                                                 /* rollout!           src/problem.jl:330-340 */
int to_expand(to_handle* h);                                                  /* RD.jacobian!(ForwardAD) on the discretized dynamics at every knot */
int to_get_dynamics_jacobians(to_handle* h, double* AB /*[B][N-1][n+m][n]: n x (n+m) col-major*/);

/* ---- kernel 2: cost + constraint + AL sweep --------------------------------------------------------- */
int to_cost(to_handle* h, double* J /*[B]*/);                                 /* cost(prob)         src/problem.jl:321, src/objective.jl:89-93 */
int to_cost_knots(to_handle* h, double* Jk /*[B][N]*/);                       /* cost! / get_J      src/objective.jl:104-110 */
int to_cost_gradient(to_handle* h, double* grad /*[B][N][n+m]*/);             /* RD.gradient!       src/cost_functions.jl:137-172 */
int to_cost_hessian(to_handle* h, double* hess /*[B][N][n+m][n+m]*/);         /* RD.hessian!        src/cost_functions.jl:212-233 (written symmetric) */
int to_eval_constraints(to_handle* h, int32_t con, double* vals /*[B][last-first+1][p]*/);      /* evaluate_constraints! src/abstract_constraint.jl:200-225 */
int to_constraint_jacobians(to_handle* h, int32_t con, double* jac /*[B][last-first+1][n+m][p]*/); /* constraint_jacobians! src/abstract_constraint.jl:236-248 */
int to_constraint_hessians(to_handle* h, int32_t con, const double* lambda /*[B][last-first+1][p], NULL = the current multipliers*/,
                           double* H /*[B][last-first+1][n+m][n+m]*/);   /* grad-constraint_jacobians! src/abstract_constraint.jl:267-280: d/dz (cz' lambda) of every knot
                                                                            (`∇jacobian!`: zero for Goal / Bound, src/constraints.jl:70-73, :767-770; second-order AD otherwise) */
int to_max_violation(to_handle* h, double* v /*[B]*/);
int to_merit(to_handle* h, double* J /*[B]*/);                                /* cost + AL penalty of the current trajectory */
int to_al_expansion(to_handle* h, double* grad /*[B][N][n+m]*/, double* hess /*[B][N][n+m][n+m]*/); /* cost expansion incl. AL terms */

/* cones (stand-alone, batched over `count` vectors of length p)  src/cones.jl */
int to_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, double* px);      /* projection!  :96-127 */
int to_grad_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, double* J);  /* grad-projection! :129-188, p x p col-major each */
int to_hess_projection(to_handle* h, int32_t cone, int32_t p, int32_t count, const double* x, const double* b, double* H); /* :201-276 */

/* ---- kernel 3 + forward pass (what Altro.jl's iLQR does with the API above) --------------------------- */
int to_backward(to_handle* h, int32_t* status /*[B] or NULL*/);               /* Riccati backward pass (needs to_expand) */
int to_forward(to_handle* h, double* J /*[B] or NULL*/, double* alpha /*[B] or NULL*/); /* closed-loop rollout + line search */
int to_ilqr_step(to_handle* h, int32_t iters);                                /* iters x (expand, backward, forward), no host sync */
int to_al_update(to_handle* h);                                               /* dual + penalty update */
int to_get_gains(to_handle* h, double* K /*[B][N-1][n_e][m]: m x n_e col-major (n_e = n unless error_state)*/, double* d /*[B][N-1][m]*/);

/* ---- solve to convergence: Altro's AL-iLQR solve!, per instance ---------------------------------------------------------------------
 * Altro 0.3 is not under the reference; the semantics are restated in DESIGN.md 5d.  Per instance, independently:
 *   start   roll out from x0 and the current controls, J = merit, rho = bp_reg_initial, counters zero.  Multipliers and penalties are KEPT
 *           (a fresh problem has lambda = 0, mu = penalty_initial): to_solve continues from whatever to_al_update / to_set_multipliers left.
 *   inner   per iteration: expansion, backward pass, line search (to_ilqr_step's iteration), then
 *             dJ = J_prev - J (AL merit), 0 and dJ_counter + 1 when the line search failed (alpha = 0);
 *             gradient = mean_k max_i |d_k,i| / (|u_k,i| + 1) with the controls after the step (Altro gradient_todorov);
 *           the inner loop converges on alpha > 0 && 0 <= dJ < cost_tol && gradient < grad_tol, and ends without converging at
 *           iterations_inner (constrained problems), iterations (all iterations together) or dJ_counter > dJ_counter_limit.
 *           A backward pass that fails at bp_reg_max ends the solve of the instance: TO_SOLVE_MAX_REGULARIZATION.
 *   outer   (constrained problems) c_max = max violation when the inner loop ended: SUCCEEDED when c_max < constraint_tolerance, else
 *           MAX_ITERATIONS when the iteration cap is reached, else MAX_ITERATIONS_OUTER after iterations_outer outer iterations, else dual
 *           update + penalty update + rho reset (to_al_update) and the next inner loop.  Inner loops use the *_intermediate tolerances except
 *           in the last allowed outer iteration (Altro set_tolerances!).
 *   no constraints: one plain iLQR loop with the final tolerances; SUCCEEDED, MAX_ITERATIONS, or UNSOLVED when it stalled (dJ_counter).
 * Shared penalties (no to_set_penalties call): the penalties are per constraint, shared by the batch, so the outer loop is batch-synchronous:
 * an instance whose inner loop has ended waits (running no kernel) until no instance is in an inner loop, and the host takes the outer step;
 * every instance in outer iteration j then sees mu_j = min(mu_0 phi^j, penalty_max), exactly as when solved alone.  The shared penalties
 * left behind are those of the batch's last outer iteration.
 * Per-instance penalties (after to_set_penalties): each instance's outer step (decision, dual update, its own penalty update, rho reset,
 * fresh merit) runs on the device in the iteration in which its inner loop ends, and it goes on without waiting for the rest of the batch.
 * The statistics, X, U, lambda, K and d are those of the shared solve (bit for bit with equal rows); afterwards instance b holds its own
 * penalties, min(mu_0 phi^(outer_b - 1), penalty_max), its own multipliers, and to_merit gives its merit at its own penalties.
 * Converged instances are retired from every solver kernel: their X, U, lambda, K, d are those of the iteration
 * they stopped at, read with the getters above.
 * Altro's summary after solve! prints these statistics: examples/Cartpole.ipynb:216-223 (ALTRO), :378-382 (iLQR), examples/Quadrotor.ipynb:374-391. */
enum to_solve_status { TO_SOLVE_UNSOLVED = 0, TO_SOLVE_SUCCEEDED = 1, TO_SOLVE_MAX_ITERATIONS = 2, TO_SOLVE_MAX_ITERATIONS_OUTER = 3,
                       TO_SOLVE_MAX_REGULARIZATION = 4 };
/* Altro 0.3 SolverOptions names; defaults (to_default_solve_options) restated from Altro, pinned by the notebooks only where noted */
typedef struct to_solve_options {
    double cost_tolerance;                  /* 1e-4 (pinned: the notebook's iLQR run stops at dJ 6.9e-5) */
    double cost_tolerance_intermediate;     /* 1e-3 (unpinned; the notebook's ALTRO run sets 1e-2) */
    double gradient_tolerance;              /* 10   (unpinned) */
    double gradient_tolerance_intermediate; /* 1    (unpinned) */
    double constraint_tolerance;            /* 1e-6 (unpinned) */
    int32_t iterations;                     /* 300  (unpinned) all iterations together */
    int32_t iterations_inner;               /* 300  (unpinned) */
    int32_t iterations_outer;               /* 30   (unpinned) */
    int32_t dJ_counter_limit;               /* 10   (unpinned) */
} to_solve_options;
int to_default_solve_options(to_solve_options* o);
/* solve!(prob): outputs [B] each, any may be NULL.  cost = the objective (not the merit) of the final trajectory; dJ, gradient = those of the
 * last iteration; c_max = the max violation when the last inner loop ended (0 without constraints).  TO_EINVAL for a non-positive
 * tolerance or cap (dJ_counter_limit may be 0). */
int to_solve(to_handle* h, const to_solve_options* o, int32_t* status, int32_t* iterations, int32_t* iterations_outer, double* cost, double* dJ,
             double* gradient, double* c_max);
/* ---- a queue of problems through the batch's slots: Altro's solve! of each problem of a list longer than the batch (DESIGN.md 5n) ------
 * Every problem shares the handle's structure (model, N, costs, constraints, time steps, solver options) and brings its own x0 and initial
 * controls, and optionally its own goal state and model parameters.  The B instances of the handle are slots: a slot whose solve stops hands
 * its results back and takes the next problem at once, on the device.  Problem p's outputs are, bit for bit, what to_solve returns for an
 * instance that starts with x0 = x0[p], controls U0[p], lambda = 0, the handle's shared penalties (to_get_penalty), the goal rows
 * to_set_goal_states(xf, goal_objective, goal_constraint) would give it and the parameter row to_set_model_params would give it; they depend
 * neither on the slot nor on the problems beside it, nor on M or B (as long as B does not change an automatic kernel choice). */
typedef struct to_queue_spec {
    int32_t M;                 /* problems, >= 1 */
    int32_t U0_shared;         /* 1: U0 is one [N-1][m] for every problem */
    const double* x0;          /* [M][n] */
    const double* U0;          /* [M][N-1][m], or [N-1][m] when U0_shared = 1 */
    const double* xf;          /* [M][n] or NULL: each problem's goal, as to_set_goal_states(xf, goal_objective, goal_constraint) */
    int32_t goal_objective;
    int32_t goal_constraint;
    const double* params;      /* [M][nparams] or NULL: each problem's model parameters, as to_set_model_params */
    int32_t nparams;
    int32_t pad;
} to_queue_spec;
/* Synchronous.  Outputs [M] each, any may be NULL: to_solve's outputs, per problem; X [M][N][n] and U [M][N-1][m] or NULL: each problem's final
 * trajectory.  On return the handle is as it was: x0, trajectories, multipliers, shared and per-instance penalties and every per-instance table.
 * The solver scratch (gains, rho, to_get_solver_state) is left unspecified, and the merit is stale, as after to_solve.  Refused before any device
 * work (TO_EINVAL / TO_EDIM, with nothing changed): M < 1; a non-finite x0, U0, xf or params entry; a parameter row to_set_model_params refuses;
 * a hybrid problem; a constrained recorded-program model, or one given xf or params; the options to_solve refuses; a per-instance table the
 * queue does not replace whose rows differ between instances (cost weights, time steps, constraint data other than the Goal values xf
 * replaces, linear cost terms other than the q that xf replaces), since the results would then depend on the slot.  TO_ENOMEM, naming the
 * size, when the device cannot hold the staged problems and their outputs: the queue is never split silently. */
int to_solve_queue(to_handle* h, const to_queue_spec* q, const to_solve_options* o, int32_t* status, int32_t* iterations, int32_t* iterations_outer,
                   double* cost, double* dJ, double* gradient, double* c_max, double* X, double* U);
/* ---- the queue with per-problem tables (DESIGN.md 5p): time steps, cost weights, constraint data, AL penalties, tracking references ------
 * Each table gives every problem its own row of one per-instance table.  Problem p's rows are what the setters write, applied in this order to
 * an instance of the handle: to_set_time_steps (the dt row; the clock is left alone), to_set_cost_weights for each cost given,
 * to_set_constraint_data for each constraint given, to_update_trajectories (Xref, Uref, start), to_set_goal_states (xf, goal_objective,
 * goal_constraint), to_set_model_params, to_set_penalties per constraint given (its entry replaces the shared penalty; the others
 * keep the shared penalties, as without a table).  Its outputs are, bit for bit, what to_solve
 * returns for an instance that starts from those rows, whatever slot it ran in, as for to_solve_queue.  So with weights and xf (or a reference),
 * each problem's q | r are derived from its own weights; weights without xf or a reference leave the linear terms as they are, as
 * to_set_cost_weights does.  Not supported: a per-problem initial time (host state no result reads), per-problem initial multipliers (problems
 * start at lambda = 0), hybrid and recorded-program models (the setters refuse these tables there). */
enum to_queue_table_kind { TO_QT_TIME_STEPS = 0, TO_QT_COST_WEIGHTS = 1, TO_QT_CONSTRAINT_DATA = 2, TO_QT_PENALTIES = 3, TO_QT_REFERENCE = 4 };
typedef struct to_queue_table {
    int32_t kind;              /* to_queue_table_kind */
    int32_t index;             /* COST_WEIGHTS: the distinct cost; CONSTRAINT_DATA, PENALTIES: the constraint; REFERENCE: start; else 0 */
    int32_t len;               /* doubles per problem (N-1, to_cost_weights_len, to_constraint_data_len, 1); REFERENCE: nref */
    int32_t pad;
    const double* rows;        /* [M][len]; REFERENCE: Xref [M][nref][n] */
    const double* rows2;       /* REFERENCE: Uref [M][nref][m]; NULL otherwise */
} to_queue_table;
/* to_solve_queue with ntables tables; to_solve_queue is this call with ntables = 0.  The handle is left as to_solve_queue leaves it, its
 * per-instance tables, clocks and closed-form Jacobian columns included.  Refused before any device work, with nothing changed (TO_EINVAL /
 * TO_EDIM, naming the table, the problem and the entry): what to_solve_queue refuses; a row the table's setter refuses (a non-finite entry,
 * dt <= 0, a non-zero H where the shared H is zero, a changed +-Inf pattern of a Bound or z_max < z_min, a NORM value < 0, a penalty <= 0,
 * nref < start + N - 1, and the costs and constraints the setters keep shared, Goal constraints included: their values come from xf); a len
 * other than the table's; an unknown kind; the same table twice; a reference together with xf and goal_objective = 1.  When the run
 * fails, the handle is restored as far as the device allows, its closed-form Jacobian columns included.  The check that per-instance tables
 * agree in every instance applies to every table the call does not replace, and not to the entries it does.  TO_ENOMEM as to_solve_queue, the staged rows and slot tables counted. */
int to_solve_queue_tables(to_handle* h, const to_queue_spec* q, const to_queue_table* tables, int32_t ntables, const to_solve_options* o,
                          int32_t* status, int32_t* iterations, int32_t* iterations_outer, double* cost, double* dJ, double* gradient, double* c_max,
                          double* X, double* U);
/* ---- Lie-group error state (SURVEY 8 f2) ------------------------------------------------------------------- */
int to_backward_algebra(const to_handle* h, int32_t* variant);             /* which arithmetic the next to_backward will use: 0 = pivot-by-pivot LDL' solve
                                                                             (riccati.cu, riccati_small.cu, lie.cu), 1 = 2 x 2 block inverse + W'K update
                                                                             (riccati_frag.cu).  Same mathematics (Altro backwardpass!); the oracle mirrors
                                                                             either so that parity tests compare like with like (DESIGN.md 4a) */
/* DIAGNOSTIC (test / tuning hook, not part of the Julia shim): which kernels the next solver calls launch, as picked from the problem's
 * shape, the options and the device (DESIGN.md 4a lists the thresholds).  choice[TO_CHOICE_COUNT]:
 *   LINESEARCH  the line search's knot loop (TO_LS_*);  COST_CACHED  1: that loop reads the costs from shared memory (0 on the generic loop);
 *   BACKWARD  the backward-pass kernel (TO_BK_*);  FASTAL  1: k_riccati holds the AL terms lane-resident (0 for the other kernels);
 *   REC_FUSED  1: the records' cost expansion reads the host-built term table (0 off the record path);  LATE_LIST  1: the later line-search
 *   passes walk the list of late instances;  INST_FORWARD / INST_BACKWARD  1: the line search / the backward pass's cost and AL reads
 *   launch their per-instance (INST) variant;  RESIDENT  k_riccati_frag warps (= instances) resident at once on this device (0 off the
 *   record path): a larger batch is pulled from the work queue after the first wave.  Reads the handle only. */
enum to_choice { TO_CHOICE_LINESEARCH = 0, TO_CHOICE_COST_CACHED = 1, TO_CHOICE_BACKWARD = 2, TO_CHOICE_FASTAL = 3, TO_CHOICE_REC_FUSED = 4,
                 TO_CHOICE_LATE_LIST = 5, TO_CHOICE_INST_FORWARD = 6, TO_CHOICE_INST_BACKWARD = 7, TO_CHOICE_RESIDENT = 8, TO_CHOICE_COUNT = 9 };
enum to_linesearch_loop { TO_LS_GENERIC = 0, TO_LS_FAST = 1, TO_LS_COMPACT = 2 };
enum to_backward_kernel { TO_BK_THREAD = 0 /* k_riccati_small */, TO_BK_WARP_MMA = 1 /* k_riccati, tensor MMA */, TO_BK_WARP_DFMA = 2 /* k_riccati, DFMA */,
                          TO_BK_FRAGMENT = 3 /* k_riccati_frag, the record path */, TO_BK_DENSE_MMA = 4 /* k_riccati_dense_mma */,
                          TO_BK_DENSE_DFMA = 5 /* k_riccati_dense */ };
int to_kernel_choice(const to_handle* h, int32_t* choice);
int to_error_state_dim(const to_handle* h, int32_t* ne);                      /* RD.errstate_dim(model): n, or n - 1 with spec.error_state */
/* RD.state_diff(model, xbar, x) of every knot against the current trajectory: Xbar [B][N][n] (host) -> dx [B][N][n_e] */
int to_state_diff(to_handle* h, const double* Xbar, double* dx);
/* error-state dynamics Jacobians [A_e B_e] = G_{k+1}' [A G_k | B] after to_expand: [B][N-1][n_e+m][n_e], n_e x (n_e+m) col-major */
int to_get_error_dynamics(to_handle* h, double* ABe);
/* error-state cost + AL expansion of every knot (Altro error_expansion!): grad [B][N][n_e+m], hess [B][N][n_e+m][n_e+m] */
int to_error_expansion(to_handle* h, double* grad, double* hess);
/* DIAGNOSTIC (not part of the Julia shim; the hot path does not use it): the cost + AL expansion that the record path's Riccati kernel
 * (to_backward_algebra = 1) read in the last backward pass, copied from doubles [192, 240) of every knot's record:
 * out [B][N][48] = g~[16] | hd[16] | Hb[4][4] in the physical order of csrc/frag_layout.cuh.  TO_ESTATE when the handle is not on the
 * record path or no backward pass has written the records' expansion yet.  to_error_expansion computes the same numbers by another
 * kernel chain and does not read the records. */
int to_get_expansion_records(to_handle* h, double* out);
int to_get_multipliers(to_handle* h, int32_t con, double* lambda /*[B][last-first+1][p]*/);
int to_set_multipliers(to_handle* h, int32_t con, const double* lambda);
/* The shared penalty of constraint con.  With per-instance penalties: to_get_penalty returns the common value while every instance holds the
 * same one, else TO_ESTATE (read them with to_get_penalties); to_set_penalty writes through to every instance, the later call winning. */
int to_get_penalty(to_handle* h, int32_t con, double* mu);
int to_set_penalty(to_handle* h, int32_t con, double mu);
/* ---- per-instance AL penalties ----------------------------------------------------------------------------------
 * Instance b weighs constraint con with its own penalty mu[b] (Altro keeps one penalty per problem).  Until the first to_set_penalties there
 * is no table and every kernel and to_solve run as before; the first call fills every instance with the shared penalty of every constraint,
 * then applies its column.  From then on to_al_update scales every instance's penalties, mu <- min(mu phi, penalty_max), as it scales the
 * shared ones, to_set_options with a new penalty_initial resets every instance's, and to_solve takes each instance's outer step on the device
 * (see to_solve).  TO_EINVAL, naming the instance, with nothing changed: an entry that is non-finite or <= 0, a constraint index out of range,
 * a hybrid problem.  A batch whose instance b holds mu_b computes, bit for bit, what instance b of a batch with to_set_penalty(mu_b) computes.
 * Multi-GPU: each rank passes its shard's entries, as for x0. */
int to_set_penalties(to_handle* h, int32_t con, const double* mu /*[B]*/);
int to_get_penalties(to_handle* h, int32_t con, double* mu /*[B]*/);          /* the shared value broadcast when none are set */
int to_get_solver_state(to_handle* h, double* rho /*[B]*/, double* dV /*[B][2]*/, double* alpha /*[B]*/, int32_t* ls_iters /*[B]*/, int32_t* bp_status /*[B]*/);

/* ---- multi-GPU / measurement plumbing --------------------------------------------------------------- */
/* device pointer to {sum_b J_b, max_b violation_b} (2 doubles) refreshed by to_reduce_merit(); the host
 * framework all-reduces it (NCCL: sum on [0], max on [1]).  SURVEY 8(e). */
int to_reduce_merit(to_handle* h);
/* Same reduction, ordered after whatever part of the last iteration is still in flight on the library's side
 * stream, and handed to `consumer_stream` (a cudaStream_t, e.g. the stream the NCCL all-reduce is issued on) through
 * an event: the handle's main stream is NOT made to wait, so the next iteration keeps overlapping (DESIGN.md 5/6). */
int to_reduce_merit_async(to_handle* h, void* consumer_stream);
int to_merit_device_ptr(to_handle* h, void** ptr);
/* per-phase device timing (CUDA events on the handle's stream) for the roofline report */
enum to_phase { TO_PHASE_EXPAND = 0, TO_PHASE_BACKWARD = 1, TO_PHASE_FORWARD = 2, TO_PHASE_LADDER = 3, TO_PHASE_ACCEPT = 4, TO_PHASE_COSTEXP = 5 /* cost + AL expansion kernel of the record / materialised-expansion paths, when it is a launch of its own */,
               TO_PHASE_LATE = 6 /* overlapped iterations: dynamics + cost expansion of the instances the late line-search trials moved (side stream) */, TO_PHASE_COUNT = 8 };
int to_set_phase_timing(to_handle* h, int enable);
int to_get_phase_times(to_handle* h, double* ms /*[TO_PHASE_COUNT] accumulated*/, int64_t* launches /*[TO_PHASE_COUNT]*/, int reset);
int64_t to_launch_count(const to_handle* h);                                  /* kernels launched by this handle so far */
int to_algorithmic_bytes(const to_handle* h, int64_t* E, int64_t* R, int64_t* F); /* per instance per iteration, SURVEY 8(d) */

#ifdef __cplusplus
}
#endif
#endif
