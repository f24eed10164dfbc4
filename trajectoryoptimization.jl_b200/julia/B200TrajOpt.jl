# B200TrajOpt.jl -- thin ccall shim over libtrajopt_b200.so (include/trajopt_b200.h).
#
# NOT RUNNABLE IN THIS REPO'S IMAGE (no Julia there); kept syntactically careful and reviewed against the header.
# It gives Julia host code (and Altro.jl) a `BatchedProblem` that is built from an ordinary
# TrajectoryOptimization.Problem and overloads the functions a solver calls on it
# (rollout!, cost, evaluate_constraints!, ... -- SURVEY.md 2.3), so the hot path runs on the GPU for a whole batch.
module B200TrajOpt

using TrajectoryOptimization
using RobotDynamics
using LinearAlgebra
using Rotations
const TO = TrajectoryOptimization
const RD = RobotDynamics

const libb200 = get(ENV, "LIBTRAJOPT_B200", "libtrajopt_b200.so")

# ---- C structs (must match include/trajopt_b200.h field for field) ------------------------------------------
struct ToCostSpec
    kind::Int32; terminal::Int32
    Q::Ptr{Float64}; R::Ptr{Float64}; H::Ptr{Float64}; q::Ptr{Float64}; r::Ptr{Float64}
    c::Float64
    w::Float64; q_ref::Ptr{Float64}; q_ind::Ptr{Int32}       # DiagonalQuatCost (kind 2), else 0 / C_NULL
    prog_len::Int32; nconst::Int32; prog::Ptr{Int32}; consts::Ptr{Float64}   # recorded program (kind 3), else 0 / C_NULL
end
struct ToConstraintSpec
    kind::Int32; first::Int32; last::Int32; sense::Int32; p::Int32; flag::Int32; ninds::Int32
    inds::Ptr{Int32}; a::Ptr{Float64}; b::Ptr{Float64}; c::Ptr{Float64}; rad::Ptr{Float64}
    val::Float64
end
struct ToDynamicsSpec         # one recorded model of a hybrid problem (to_dynamics_spec; models given as programs: Python host API only for now)
    n_in::Int32; m_in::Int32; n_out::Int32; discrete::Int32; prog_len::Int32; nconst::Int32
    prog::Ptr{Int32}; consts::Ptr{Float64}
end
struct ToSpec
    model::Int32; n::Int32; m::Int32; N::Int32; B::Int32; device::Int32; nparams::Int32
    params::Ptr{Float64}; dt::Ptr{Float64}; t0::Float64
    ncost::Int32; costs::Ptr{ToCostSpec}; cost_index::Ptr{Int32}
    ncon::Int32; cons::Ptr{ToConstraintSpec}
    error_state::Int32       # 1: solver kernels on the Lie-group error state (RD.errstate_dim(model) != n), as Altro does
    ndyn::Int32; dyn::Ptr{ToDynamicsSpec}; dyn_index::Ptr{Int32}; nx::Ptr{Int32}; nu::Ptr{Int32}    # TO_MODEL_EXPR only, else 0 / C_NULL
end

const TO_EDIM = -2
const TO_EINVAL = -1

function check(h::Ptr{Cvoid}, rc::Cint)
    rc == 0 && return nothing
    msg = unsafe_string(ccall((:to_last_error, libb200), Cstring, (Ptr{Cvoid},), h))
    rc == TO_EDIM && throw(DimensionMismatch(msg))     # same exception types as src/problem.jl:64-68, :87-91
    rc == TO_EINVAL && throw(ArgumentError(msg))
    error("libtrajopt_b200 [$rc]: $msg")
end

"""
    recorded_dims(nx_max, nu_max) -> (n, m)

The padded size class a problem of recorded dynamics programs (`TO_MODEL_EXPR`) runs on: the smallest of (4, 2), (8, 4) and (16, 8) that
holds its largest per-knot state dimension `nx_max` and control dimension `nu_max` (`RD.dims(models)`).  `ToSpec.n, m` of such a problem
must be this class; `DimensionMismatch` past 16 states or 8 controls.
"""
function recorded_dims(nx_max::Integer, nu_max::Integer)
    n = Ref{Int32}(0); m = Ref{Int32}(0)
    rc = ccall((:to_recorded_dims, libb200), Cint, (Int32, Int32, Ref{Int32}, Ref{Int32}), nx_max, nu_max, n, m)
    rc == TO_EDIM && throw(DimensionMismatch("recorded-program models: at most 16 states and 8 controls per knot, the largest has ($nx_max, $nu_max)"))
    rc == 0 || throw(ArgumentError("recorded-program models: no size class for ($nx_max, $nu_max)"))
    (Int(n[]), Int(m[]))
end

model_id(::Any) = error("model not available on the device; supported: DoubleIntegrator, Cartpole, Quadrotor, Acrobot")

mutable struct BatchedProblem
    h::Ptr{Cvoid}
    prob::TO.Problem          # the template instance (objective / constraint objects stay the reference's)
    B::Int
    keep::Vector{Any}         # GC roots of every array whose pointer went into the spec
end

sense_code(::TO.Equality) = Int32(0)
sense_code(::TO.Inequality) = Int32(1)
sense_code(::TO.SecondOrderCone) = Int32(2)
sense_code(::TO.IdentityCone) = Int32(3)
sense_code(::TO.PositiveOrthant) = Int32(4)

# ---- ConstraintList entry -> to_constraint_spec (include/trajopt_b200.h to_con_kind), every constraint type of src/constraints.jl ----
# `root` keeps the arrays whose pointers go into the spec alive until to_create has copied them.
const NULLI = Ptr{Int32}(C_NULL); const NULLD = Ptr{Float64}(C_NULL)
function constraint_spec(con::TO.GoalConstraint, f, l, n, m, root)                    # src/constraints.jl:22-87
    ii = root(Vector{Int32}(con.inds)); a = root(Vector{Float64}(con.xf))
    ToConstraintSpec(0, f, l, 0, 0, 0, length(ii), pointer(ii), pointer(a), NULLD, NULLD, NULLD, 0.0)
end
function constraint_spec(con::TO.BoundConstraint, f, l, n, m, root)                   # :644-783
    a = root(Vector{Float64}(con.z_max)); b = root(Vector{Float64}(con.z_min))
    ToConstraintSpec(1, f, l, 1, 0, 0, 0, NULLI, pointer(a), pointer(b), NULLD, NULLD, 0.0)
end
function bound_base_spec(bnd, f, l, n, m, root, control::Bool)                        # StateBound / ControlBound :547-631 = Bound with the other block open
    zmax = fill(Inf, n + m); zmin = fill(-Inf, n + m); off = control ? n : 0
    zmax[off .+ bnd.i_max] .= bnd.x_max; zmin[off .+ bnd.i_min] .= bnd.x_min
    a = root(zmax); b = root(zmin)
    ToConstraintSpec(1, f, l, 1, 0, 0, 0, NULLI, pointer(a), pointer(b), NULLD, NULLD, 0.0)
end
constraint_spec(con::TO.StateBound, f, l, n, m, root) = bound_base_spec(con.bnd, f, l, n, m, root, false)
constraint_spec(con::TO.ControlBound, f, l, n, m, root) = bound_base_spec(con.bnd, f, l, n, m, root, true)
function constraint_spec(con::TO.LinearConstraint, f, l, n, m, root)                  # :103-150 -- A acts on z[inds]; the device takes the x or the u block
    inds = collect(con.inds); P = length(con.b)
    A = Matrix{Float64}(con.A)
    if all(i -> i <= n, inds)
        Af = zeros(P, n); Af[:, inds] .= A; flag = 0
    elseif all(i -> i > n, inds)
        Af = zeros(P, m); Af[:, inds .- n] .= A; flag = 1
    else
        throw(ArgumentError("LinearConstraint across states and controls: split it into a state and a control constraint for the device"))
    end
    a = root(Af); b = root(Vector{Float64}(con.b))                                     # column-major p x w, as the ABI wants
    ToConstraintSpec(2, f, l, sense_code(con.sense), P, flag, 0, NULLI, pointer(a), pointer(b), NULLD, NULLD, 0.0)
end
function constraint_spec(con::TO.CircleConstraint, f, l, n, m, root)                  # :168-233
    a = root(Vector{Float64}(con.x)); b = root(Vector{Float64}(con.y)); r = root(Vector{Float64}(con.radius))
    ii = root(Int32[con.xi, con.yi])
    ToConstraintSpec(3, f, l, 1, length(a), 0, 2, pointer(ii), pointer(a), pointer(b), NULLD, pointer(r), 0.0)
end
function constraint_spec(con::TO.SphereConstraint, f, l, n, m, root)                  # :249-326
    a = root(Vector{Float64}(con.x)); b = root(Vector{Float64}(con.y)); c = root(Vector{Float64}(con.z)); r = root(Vector{Float64}(con.radius))
    ii = root(Int32[con.xi, con.yi, con.zi])
    ToConstraintSpec(4, f, l, 1, length(a), 0, 3, pointer(ii), pointer(a), pointer(b), pointer(c), pointer(r), 0.0)
end
function constraint_spec(con::TO.NormConstraint, f, l, n, m, root)                    # :438-521 (the static evaluate: z[inds[j]], SURVEY 2.4)
    ii = root(Vector{Int32}(con.inds))
    ToConstraintSpec(5, f, l, sense_code(con.sense), 0, 0, length(ii), pointer(ii), NULLD, NULLD, NULLD, NULLD, Float64(con.val))
end
function constraint_spec(con::TO.CollisionConstraint, f, l, n, m, root)               # :341-389
    ii = root(Int32[con.x1; con.x2])
    ToConstraintSpec(6, f, l, 1, 0, 0, length(ii), pointer(ii), NULLD, NULLD, NULLD, NULLD, con.radius)
end
function constraint_spec(con::TO.QuatVecEq, f, l, n, m, root)                         # :938-965
    a = root(Vector{Float64}(Rotations.params(con.qf))); ii = root(Vector{Int32}(con.qind))
    ToConstraintSpec(7, f, l, 0, 3, 0, 4, pointer(ii), pointer(a), NULLD, NULLD, NULLD, 0.0)
end
function constraint_spec(con::TO.IndexedConstraint, f, l, n, m, root)                 # :820-936: the inner constraint with its indices moved into the new z
    ix, iu = collect(con.ix), collect(con.iu) .- con.n                                # positions of the old x / u inside the new x / u
    constraint_spec(TO.change_dimension(con.con, n, m, ix, iu), f, l, n, m, root)
end
function constraint_spec(con::TO.StageConstraint, f, l, n, m, root)                   # RD.@autodiff user constraint: record RD.evaluate
    tape = root(record((x, u) -> RD.evaluate(con, x, u), n, m))
    P = RD.output_dim(con)
    ToConstraintSpec(8, f, l, sense_code(TO.sense(con)), P, length(tape.consts), length(tape.prog), pointer(tape.prog), pointer(tape.consts), NULLD, NULLD, NULLD, 0.0)
end

# the to_integration code of an explicit RobotDynamics rule; the implicit rules are refused (iLQR's rollout needs an explicit step)
integration_code(::RD.Euler) = Int32(1)
integration_code(::RD.RK2) = Int32(2)
integration_code(::RD.RK3) = Int32(3)
integration_code(::RD.RK4) = Int32(4)
integration_code(rule) = throw(ArgumentError("integration $(typeof(rule)) is not supported: the explicit rules RD.Euler, RD.RK2, RD.RK3 and RD.RK4 are"))

"""
    BatchedProblem(prob::TO.Problem, model_id, B; device=0, params=Float64[], integration=RD.integration(prob.model[1]))

Describe `prob` (objective = vector of QuadraticCostFunctions, ConstraintList of Goal/Bound/Linear/Circle/Sphere/Norm)
to the library and allocate a batch of `B` instances on `device`.  `integration` is the explicit rule the dynamics are discretised
with (to_set_integration): `prob`'s own by default.
"""
function BatchedProblem(prob::TO.Problem, mid::Integer, B::Integer; device::Integer=0, params::Vector{Float64}=Float64[],
                        error_state::Bool=(RD.errstate_dim(TO.get_model(prob)[1]) != RD.state_dim(TO.get_model(prob)[1])),
                        integration=RD.integration(TO.get_model(prob)[1]))
    rule = integration_code(integration)
    n, m, N = RD.dims(prob, 1)
    keep = Any[]
    root(x) = (push!(keep, x); x)
    obj = TO.get_objective(prob)
    costs = ToCostSpec[]
    index = Int32[]
    seen = IdDict{Any,Int32}()
    for k = 1:N
        c = obj[k]
        if !haskey(seen, c) && !(c isa TO.QuadraticCostFunction)      # RD.@autodiff user cost: record RD.evaluate
            tape = root(record((x, u) -> RD.evaluate(c, x, u), n, m))
            push!(costs, expr_cost_spec(tape, k == N))
            seen[c] = Int32(length(costs) - 1)
        elseif !haskey(seen, c)
            isdiag = TO.is_diag(c)
            Q = root(isdiag ? Vector{Float64}(diag(c.Q)) : Matrix{Float64}(c.Q))
            R = root(isdiag ? Vector{Float64}(diag(c.R)) : Matrix{Float64}(c.R))
            H = isdiag ? C_NULL : pointer(root(Matrix{Float64}(c.H)))
            q = root(Vector{Float64}(c.q)); r = root(Vector{Float64}(c.r))
            if c isa TO.DiagonalQuatCost                         # src/lie_costs.jl:33-56
                qref = root(Vector{Float64}(c.q_ref)); qind = root(Vector{Int32}(c.q_ind))
                push!(costs, ToCostSpec(2, c.terminal ? 1 : 0, pointer(Q), pointer(R), C_NULL, pointer(q), pointer(r), c.c, c.w, pointer(qref), pointer(qind), 0, 0, C_NULL, C_NULL))
            else
                push!(costs, ToCostSpec(isdiag ? 0 : 1, c.terminal ? 1 : 0, pointer(Q), pointer(R), H, pointer(q), pointer(r), c.c, 0.0, C_NULL, C_NULL, 0, 0, C_NULL, C_NULL))
            end
            seen[c] = Int32(length(costs) - 1)
        end
        push!(index, seen[c])
    end
    cons = ToConstraintSpec[]
    for (inds, con) in zip(TO.get_constraints(prob))
        f, l = Int32(first(inds)), Int32(last(inds))
        push!(cons, constraint_spec(con, f, l, n, m, root))
    end
    dt = root(Vector{Float64}([RD.timestep(z) for z in TO.get_trajectory(prob)][1:N-1]))
    root(costs); root(index); root(cons); root(params)
    spec = Ref(ToSpec(mid, n, m, N, B, device, length(params), isempty(params) ? C_NULL : pointer(params), pointer(dt),
                      TO.get_initial_time(prob), length(costs), pointer(costs), pointer(index), length(cons),
                      isempty(cons) ? C_NULL : pointer(cons), error_state ? 1 : 0, 0, C_NULL, C_NULL, C_NULL, C_NULL))
    h = Ref{Ptr{Cvoid}}(C_NULL)
    rc = GC.@preserve keep ccall((:to_create, libb200), Cint, (Ref{ToSpec}, Ref{Ptr{Cvoid}}), spec, h)
    check(C_NULL, rc)
    bp = BatchedProblem(h[], prob, B, keep)
    finalizer(p -> ccall((:to_destroy, libb200), Cint, (Ptr{Cvoid},), p.h), bp)
    check(bp.h, ccall((:to_set_integration, libb200), Cint, (Ptr{Cvoid}, Int32), bp.h, rule))
    return bp
end

# ---- user-defined costs / constraints (RD.@autodiff types): record RD.evaluate once, ship the tape ---------------------
# The device differentiates a straight-line program with second-order forward-mode duals (include/trajopt_b200.h to_expr_op).
# `Rec` is a number type that appends one instruction per arithmetic operation -- the trick ForwardDiff.Dual uses to see the
# user's function, applied to recording instead of differentiating.
mutable struct Tape
    prog::Vector{Int32}      # op, a, b triples (0-based operand indices)
    consts::Vector{Float64}
end
Tape() = Tape(Int32[], Float64[])
struct Rec <: Real
    tape::Tape
    idx::Int32               # 0-based index of the instruction that produced this value
end
function emit!(t::Tape, op, a, b)
    push!(t.prog, Int32(op), Int32(a), Int32(b))
    Rec(t, Int32(length(t.prog) ÷ 3 - 1))
end
function constindex!(t::Tape, v::Real)
    i = findfirst(c -> c === Float64(v), t.consts)
    i === nothing ? (push!(t.consts, Float64(v)); length(t.consts) - 1) : i - 1
end
Base.promote_rule(::Type{Rec}, ::Type{<:Real}) = Rec
for (f, op, opc, ropc) in ((:+, 3, 15, 15), (:*, 5, 16, 16))             # commutative: ADD / ADDC, MUL / MULC
    @eval Base.$f(a::Rec, b::Rec) = emit!(a.tape, $op, a.idx, b.idx)
    @eval Base.$f(a::Rec, b::Real) = emit!(a.tape, $opc, a.idx, constindex!(a.tape, b))
    @eval Base.$f(a::Real, b::Rec) = emit!(b.tape, $ropc, b.idx, constindex!(b.tape, a))
end
Base.:-(a::Rec, b::Rec) = emit!(a.tape, 4, a.idx, b.idx)
Base.:-(a::Rec, b::Real) = emit!(a.tape, 15, a.idx, constindex!(a.tape, -b))    # a + (-b)
Base.:-(a::Real, b::Rec) = emit!(b.tape, 19, b.idx, constindex!(b.tape, a))     # RSUBC
Base.:-(a::Rec) = emit!(a.tape, 7, a.idx, 0)
Base.:/(a::Rec, b::Rec) = emit!(a.tape, 6, a.idx, b.idx)
Base.:/(a::Rec, b::Real) = emit!(a.tape, 17, a.idx, constindex!(a.tape, b))     # DIVC
Base.:/(a::Real, b::Rec) = emit!(b.tape, 18, b.idx, constindex!(b.tape, a))     # RDIVC
Base.:^(a::Rec, p::Integer) = p == 2 ? a * a : emit!(a.tape, 13, a.idx, constindex!(a.tape, p))
Base.:^(a::Rec, p::Real) = emit!(a.tape, 13, a.idx, constindex!(a.tape, p))     # POWC
for (f, op) in ((:sin, 8), (:cos, 9), (:exp, 10), (:log, 11), (:sqrt, 12), (:tanh, 14))
    @eval Base.$f(a::Rec) = emit!(a.tape, $op, a.idx, 0)
end

"""
    record(f, n, m) -> Tape

Call `f(x, u)` (e.g. `(x, u) -> RD.evaluate(cost, x, u)`) on recording vectors and return the tape; the last instruction is the
value (scalar costs) or the last `p` instructions are the outputs (constraints: `f` returns a vector, each entry is re-emitted).
"""
function record(f, n::Integer, m::Integer)
    t = Tape()
    x = [emit!(t, 1, i - 1, 0) for i = 1:n]          # TO_OP_X
    u = [emit!(t, 2, j - 1, 0) for j = 1:m]          # TO_OP_U
    out = f(x, u)
    for o in (out isa AbstractVector ? out : (out,))
        o isa Rec ? emit!(t, 15, o.idx, constindex!(t, 0.0)) : emit!(t, 0, constindex!(t, o), 0)
    end
    return t
end
expr_cost_spec(t::Tape, terminal::Bool) =            # ToCostSpec of kind TO_COST_EXPR (keep `t` alive: GC roots)
    ToCostSpec(3, terminal ? 1 : 0, C_NULL, C_NULL, C_NULL, C_NULL, C_NULL, 0.0, 0.0, C_NULL, C_NULL,
               Int32(length(t.prog) ÷ 3), Int32(length(t.consts)), pointer(t.prog), pointer(t.consts))

# ---- the operator surface a solver calls (SURVEY.md 2.3) ------------------------------------------------------
# host arrays are Array{Float64,3}: X (n, N, B), U (m, N-1, B) -- exactly the library's instance-major layout.
TO.set_initial_state!(p::BatchedProblem, x0::Matrix{Float64}) =          # src/problem.jl:270
    check(p.h, ccall((:to_set_initial_state, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, x0))
TO.initial_controls!(p::BatchedProblem, U::Array{Float64,3}) =           # src/problem.jl:261
    check(p.h, ccall((:to_set_controls, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, U))
TO.initial_states!(p::BatchedProblem, X::Array{Float64,3}) =             # src/problem.jl:253
    check(p.h, ccall((:to_set_states, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, X))
TO.rollout!(p::BatchedProblem) =                                         # src/problem.jl:330-340
    check(p.h, ccall((:to_rollout, libb200), Cint, (Ptr{Cvoid},), p.h))
function TO.cost(p::BatchedProblem)                                      # src/problem.jl:321
    J = Vector{Float64}(undef, p.B)
    check(p.h, ccall((:to_cost, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, J)); J
end
function TO.states(p::BatchedProblem)                                    # src/problem.jl:175
    n, m, N = RD.dims(p.prob, 1); X = Array{Float64,3}(undef, n, N, p.B)
    check(p.h, ccall((:to_get_states, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, X)); X
end
function TO.controls(p::BatchedProblem)                                  # src/problem.jl:168
    n, m, N = RD.dims(p.prob, 1); U = Array{Float64,3}(undef, m, N - 1, p.B)
    check(p.h, ccall((:to_get_controls, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, U)); U
end
function TO.evaluate_constraints!(p::BatchedProblem, con_index::Integer, vals::Array{Float64,3})   # src/abstract_constraint.jl:200-225
    check(p.h, ccall((:to_eval_constraints, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con_index - 1, vals)); vals
end
function TO.constraint_jacobians!(p::BatchedProblem, con_index::Integer, jac::Array{Float64,4})    # src/abstract_constraint.jl:236-248
    check(p.h, ccall((:to_constraint_jacobians, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con_index - 1, jac)); jac
end

# ---- the same sweeps with the REFERENCE'S OWN SIGNATURES (src/abstract_constraint.jl:200-280), dispatching on a batched trajectory ----
# Altro calls   evaluate_constraints!(sig, con, vals, Z, inds) / constraint_jacobians!(sig, dif, con, jac, vals, Z, inds)
# with Z = get_trajectory(prob).  `get_trajectory(::BatchedProblem)` returns a BatchedTrajectory, so those calls land here unchanged; the
# output containers are 3- / 4-dimensional arrays (p, length(inds), B) / (p, n+m, length(inds), B) instead of vectors of vectors.
struct BatchedTrajectory
    p::BatchedProblem
end
TO.get_trajectory(p::BatchedProblem) = BatchedTrajectory(p)
function con_index(p::BatchedProblem, con, inds)
    for (i, (ii, c)) in enumerate(zip(TO.get_constraints(p.prob)))
        c === con && first(ii) == first(inds) && last(ii) == last(inds) && return i
    end
    throw(ArgumentError("constraint / knot range is not part of the batched problem's ConstraintList"))
end
TO.evaluate_constraints!(::RD.FunctionSignature, con::TO.StageConstraint, vals::Array{Float64,3}, Z::BatchedTrajectory, inds) =
    TO.evaluate_constraints!(Z.p, con_index(Z.p, con, inds), vals)
TO.constraint_jacobians!(::RD.FunctionSignature, ::RD.DiffMethod, con::TO.StageConstraint, jac::Array{Float64,4}, vals, Z::BatchedTrajectory, inds) =
    TO.constraint_jacobians!(Z.p, con_index(Z.p, con, inds), jac)
# second-order term: H[:, :, j, b] = d/dz (grad c' lambda) at knot inds[j] of instance b  (to_constraint_hessians; lambda = (p, length(inds), B) or nothing = the current multipliers)
function TO.∇constraint_jacobians!(::RD.FunctionSignature, ::RD.DiffMethod, con::TO.StageConstraint, H::Array{Float64,4}, λ, vals, Z::BatchedTrajectory, inds)
    lp = λ === nothing ? Ptr{Float64}(C_NULL) : pointer(λ)
    GC.@preserve λ check(Z.p.h, ccall((:to_constraint_hessians, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}, Ptr{Float64}), Z.p.h, con_index(Z.p, con, inds) - 1, lp, H))
    H
end
# cost expansion of every knot of every instance: RD.gradient!(cost, grad, z) / RD.hessian!(cost, hess, z)  (src/cost_functions.jl:137-233)
function RD.gradient!(p::BatchedProblem, grad::Array{Float64,3})            # (n+m, N, B)
    check(p.h, ccall((:to_cost_gradient, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, grad)); grad
end
function RD.hessian!(p::BatchedProblem, hess::Array{Float64,4})             # (n+m, n+m, N, B), written symmetric
    check(p.h, ccall((:to_cost_hessian, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, hess)); hess
end
function TO.cost!(p::BatchedProblem, J::Matrix{Float64})                    # cost!(obj, Z) src/objective.jl:104-106: (N, B) knot costs
    check(p.h, ccall((:to_cost_knots, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, J)); J
end
# cones (src/cones.jl:71-276) on `count` vectors of length p at once: x, px (p, count); J, H (p, p, count)
TO.projection!(p::BatchedProblem, cone::TO.ConstraintSense, px::Matrix{Float64}, x::Matrix{Float64}) =
    (check(p.h, ccall((:to_projection, libb200), Cint, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Float64}, Ptr{Float64}), p.h, sense_code(cone), size(x, 1), size(x, 2), x, px)); px)
TO.∇projection!(p::BatchedProblem, cone::TO.ConstraintSense, J::Array{Float64,3}, x::Matrix{Float64}) =
    (check(p.h, ccall((:to_grad_projection, libb200), Cint, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Float64}, Ptr{Float64}), p.h, sense_code(cone), size(x, 1), size(x, 2), x, J)); J)
TO.∇²projection!(p::BatchedProblem, cone::TO.ConstraintSense, H::Array{Float64,3}, x::Matrix{Float64}, b::Matrix{Float64}) =
    (check(p.h, ccall((:to_hess_projection, libb200), Cint, (Ptr{Cvoid}, Int32, Int32, Int32, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}), p.h, sense_code(cone), size(x, 1), size(x, 2), x, b, H)); H)

TO.set_goal_state!(p::BatchedProblem, xf::Vector{Float64}; objective=true, constraint=true) =      # src/problem.jl:294-310
    check(p.h, ccall((:to_set_goal_state, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint, Cint), p.h, xf, objective, constraint))
# per instance: column b of xf (n, B) is instance b's goal (its own q = -Q xf_b and Goal values; Q, R, c and the rest stay shared)
function TO.set_goal_state!(p::BatchedProblem, xf::AbstractMatrix{Float64}; objective=true, constraint=true)
    size(xf, 2) == p.B || throw(DimensionMismatch("xf must be (n, B)"))
    check(p.h, ccall((:to_set_goal_states, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Cint, Cint), p.h, Matrix{Float64}(xf), objective, constraint))
end
# per-instance model parameters: column b of P (nparams, B) is instance b's parameter vector, in the order of to_spec.params
function set_model_params!(p::BatchedProblem, P::AbstractMatrix)
    size(P, 2) == p.B || throw(DimensionMismatch("P must be (nparams, B)"))
    check(p.h, ccall((:to_set_model_params, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Int32), p.h, Matrix{Float64}(P), size(P, 1)))
end
function model_params(p::BatchedProblem, nparams::Integer)
    P = Matrix{Float64}(undef, nparams, p.B)
    check(p.h, ccall((:to_get_model_params, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, P))
    P
end
# per-instance time steps: column b of dt (N-1, B) is instance b's steps, t0[b] its initial time (nothing: keep the clocks)
function set_time_steps!(p::BatchedProblem, dt::AbstractMatrix, t0::Union{Nothing,AbstractVector}=nothing)
    size(dt) == (p.prob.N - 1, p.B) || throw(DimensionMismatch("dt must be (N-1, B)"))
    t0 === nothing || length(t0) == p.B || throw(DimensionMismatch("t0 must have length B"))
    check(p.h, ccall((:to_set_time_steps, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), p.h, Matrix{Float64}(dt),
                     t0 === nothing ? C_NULL : Vector{Float64}(t0)))
end
set_time_steps!(p::BatchedProblem, dt::AbstractVector, t0=nothing) = set_time_steps!(p, repeat(permutedims(Vector{Float64}(dt)), p.prob.N - 1), t0)
# RD.integration(prob.model[1]) of the batch: the code of its explicit rule (1 Euler, 2 RK2, 3 RK3, 4 RK4)
function integration(p::BatchedProblem)
    rule = Ref{Int32}(0)
    check(p.h, ccall((:to_get_integration, libb200), Cint, (Ptr{Cvoid}, Ref{Int32}), p.h, rule))
    return rule[]
end

function time_steps(p::BatchedProblem)
    dt = Matrix{Float64}(undef, p.prob.N - 1, p.B)
    t0 = Vector{Float64}(undef, p.B)
    check(p.h, ccall((:to_get_time_steps, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), p.h, dt, t0))
    dt, t0
end
# per-instance constraint data: column b of D (len, B) is instance b's data of constraint `con` (1-based), in the layout of
# to_set_constraint_data (Bound z_max | z_min, Linear b, Circle xc | yc | r, Sphere xc | yc | zc | r, Norm val, Collision radius)
function constraint_data_len(p::BatchedProblem, con::Integer)
    len = Ref{Int32}(0)
    check(p.h, ccall((:to_constraint_data_len, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Int32}), p.h, con - 1, len))
    Int(len[])
end
function set_constraint_data!(p::BatchedProblem, con::Integer, D::AbstractMatrix)
    size(D) == (constraint_data_len(p, con), p.B) || throw(DimensionMismatch("D must be (len, B)"))
    check(p.h, ccall((:to_set_constraint_data, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con - 1, Matrix{Float64}(D)))
end
function constraint_data(p::BatchedProblem, con::Integer)
    D = Matrix{Float64}(undef, constraint_data_len(p, con), p.B)
    check(p.h, ccall((:to_get_constraint_data, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con - 1, D))
    D
end
# per-instance cost weights: column b of W (len, B) is instance b's weights of distinct cost `cost` (1-based), in the layout of
# to_set_cost_weights (DiagonalCost Qd | Rd | c, QuadraticCost Q | R | H | c column-major, DiagonalQuatCost Qd | Rd | c | w)
function cost_weights_len(p::BatchedProblem, cost::Integer)
    len = Ref{Int32}(0)
    check(p.h, ccall((:to_cost_weights_len, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Int32}), p.h, cost - 1, len))
    Int(len[])
end
function set_cost_weights!(p::BatchedProblem, cost::Integer, W::AbstractMatrix)
    size(W) == (cost_weights_len(p, cost), p.B) || throw(DimensionMismatch("W must be (len, B)"))
    check(p.h, ccall((:to_set_cost_weights, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, cost - 1, Matrix{Float64}(W)))
end
function cost_weights(p::BatchedProblem, cost::Integer)
    W = Matrix{Float64}(undef, cost_weights_len(p, cost), p.B)
    check(p.h, ccall((:to_get_cost_weights, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, cost - 1, W))
    W
end
# per-instance AL penalties: mu[b] is instance b's penalty of constraint `con` (1-based); a scalar sets every instance's
function set_penalties!(p::BatchedProblem, con::Integer, mu::AbstractVector)
    length(mu) == p.B || throw(DimensionMismatch("mu must have length B"))
    check(p.h, ccall((:to_set_penalties, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con - 1, Vector{Float64}(mu)))
end
set_penalties!(p::BatchedProblem, con::Integer, mu::Real) = set_penalties!(p, con, fill(Float64(mu), p.B))
function penalties(p::BatchedProblem, con::Integer)
    mu = Vector{Float64}(undef, p.B)
    check(p.h, ccall((:to_get_penalties, libb200), Cint, (Ptr{Cvoid}, Int32, Ptr{Float64}), p.h, con - 1, mu))
    mu
end

# ---- what Altro.jl's iLQR / AL loop does with the API above, fused on the device ------------------------------
expand!(p::BatchedProblem) = check(p.h, ccall((:to_expand, libb200), Cint, (Ptr{Cvoid},), p.h))
backwardpass!(p::BatchedProblem) = check(p.h, ccall((:to_backward, libb200), Cint, (Ptr{Cvoid}, Ptr{Int32}), p.h, C_NULL))
forwardpass!(p::BatchedProblem) = check(p.h, ccall((:to_forward, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}), p.h, C_NULL, C_NULL))
ilqr_step!(p::BatchedProblem, iters::Integer=1) = check(p.h, ccall((:to_ilqr_step, libb200), Cint, (Ptr{Cvoid}, Int32), p.h, iters))
al_update!(p::BatchedProblem) = check(p.h, ccall((:to_al_update, libb200), Cint, (Ptr{Cvoid},), p.h))
function max_violation(p::BatchedProblem)
    v = Vector{Float64}(undef, p.B)
    check(p.h, ccall((:to_max_violation, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}), p.h, v)); v
end

# Altro's AL-iLQR solve!, per instance, on the device (to_solve; include/trajopt_b200.h, DESIGN.md 5d).  Keywords: Altro 0.3 SolverOptions
# names (cost_tolerance, cost_tolerance_intermediate, gradient_tolerance, gradient_tolerance_intermediate, constraint_tolerance, iterations,
# iterations_inner, iterations_outer, dJ_counter_limit).  Returns the per-instance summary Altro prints after solve!
# (examples/Cartpole.ipynb:216-223, :378-382); the trajectories stay in the problem (states / controls / multipliers getters).
struct ToSolveOptions
    cost_tolerance::Float64
    cost_tolerance_intermediate::Float64
    gradient_tolerance::Float64
    gradient_tolerance_intermediate::Float64
    constraint_tolerance::Float64
    iterations::Int32
    iterations_inner::Int32
    iterations_outer::Int32
    dJ_counter_limit::Int32
end
const SOLVE_STATUS = (:UNSOLVED, :SOLVE_SUCCEEDED, :MAX_ITERATIONS, :MAX_ITERATIONS_OUTER, :MAX_REGULARIZATION)   # to_solve_status 0..4
# Altro's defaults (to_default_solve_options) with the keyword overrides
function solve_options(kw)
    d = Ref{ToSolveOptions}()
    ccall((:to_default_solve_options, libb200), Cint, (Ref{ToSolveOptions},), d)
    vals = Dict{Symbol,Any}(f => getfield(d[], f) for f in fieldnames(ToSolveOptions))
    for (k, v) in kw
        haskey(vals, k) || throw(ArgumentError("unknown solve option $k"))
        vals[k] = v
    end
    Ref(ToSolveOptions((convert(fieldtype(ToSolveOptions, f), vals[f]) for f in fieldnames(ToSolveOptions))...))
end
function solve!(p::BatchedProblem; kw...)
    o = solve_options(kw)
    status, iters, outer = Vector{Int32}(undef, p.B), Vector{Int32}(undef, p.B), Vector{Int32}(undef, p.B)
    cost, dJ, grad, cmax = (Vector{Float64}(undef, p.B) for _ in 1:4)
    check(p.h, ccall((:to_solve, libb200), Cint,
                     (Ptr{Cvoid}, Ref{ToSolveOptions}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                     p.h, o, status, iters, outer, cost, dJ, grad, cmax))
    (status = [SOLVE_STATUS[s + 1] for s in status], iterations = iters, iterations_outer = outer, cost = cost, dJ = dJ, gradient = grad, c_max = cmax)
end

# a queue of M problems through the batch's slots (to_solve_queue, DESIGN.md 5n): Altro's loop of solve! over many Problems, on the device.
# x0s (n, M); U0s (m, N-1, M) or (m, N-1) for every problem; xf (n, M) or nothing (objective / constraint as set_goal_state!); params
# (nparams, M) or nothing.  A named tuple of [M] vectors as solve! returns, plus X (n, N, M) and U (m, N-1, M).
struct ToQueueSpec
    M::Int32; U0_shared::Int32
    x0::Ptr{Float64}; U0::Ptr{Float64}; xf::Ptr{Float64}
    goal_objective::Int32; goal_constraint::Int32
    params::Ptr{Float64}
    nparams::Int32; pad::Int32
end
# Per-problem tables (to_solve_queue_tables, DESIGN.md 5p), each as its setter takes it with M columns: dt (N-1, M); cost_weights and
# constraint_data Dicts of the (1-based) distinct cost / constraint => (len, M); penalties a Dict of the (1-based) constraint => mu (M),
# the others keeping the shared penalty; Xref (n, nref, M) with Uref (m, nref, M) and start.  Problem p's rows are those the setters write in the order of the C header.
struct ToQueueTable
    kind::Int32; index::Int32; len::Int32; pad::Int32
    rows::Ptr{Float64}; rows2::Ptr{Float64}
end
function solve_queue!(p::BatchedProblem, x0s, U0s; xf = nothing, params = nothing, objective::Bool = true, constraint::Bool = true,
                      dt = nothing, cost_weights = Dict(), constraint_data = Dict(), penalties = Dict(), Xref = nothing, Uref = nothing,
                      start::Integer = 1, kw...)
    X0 = Matrix{Float64}(x0s); M = size(X0, 2)
    U0 = Array{Float64}(U0s); shared = ndims(U0) == 2
    (shared || size(U0, 3) == M) || throw(DimensionMismatch("U0s must be (m, N-1, M) or (m, N-1)"))
    XF = xf === nothing ? nothing : Matrix{Float64}(xf)
    XF === nothing || size(XF, 2) == M || throw(DimensionMismatch("xf must be (n, M)"))
    P = params === nothing ? nothing : Matrix{Float64}(params)
    P === nothing || size(P, 2) == M || throw(DimensionMismatch("params must be (nparams, M)"))
    (Xref === nothing) == (Uref === nothing) || throw(ArgumentError("Xref and Uref come together"))
    o = solve_options(kw)
    n, N = size(X0, 1), size(U0, 2) + 1; m = size(U0, 1)
    keep = Any[]      # the arrays the tables point into
    tables = ToQueueTable[]
    if dt !== nothing
        D = Matrix{Float64}(dt); size(D) == (N - 1, M) || throw(DimensionMismatch("dt must be (N-1, M)"))
        push!(keep, D); push!(tables, ToQueueTable(0, 0, N - 1, 0, pointer(D), C_NULL))
    end
    for (c, W) in cost_weights
        A = Matrix{Float64}(W); size(A, 2) == M || throw(DimensionMismatch("cost weights must be (len, M)"))
        push!(keep, A); push!(tables, ToQueueTable(1, c - 1, size(A, 1), 0, pointer(A), C_NULL))
    end
    for (c, W) in constraint_data
        A = Matrix{Float64}(W); size(A, 2) == M || throw(DimensionMismatch("constraint data must be (len, M)"))
        push!(keep, A); push!(tables, ToQueueTable(2, c - 1, size(A, 1), 0, pointer(A), C_NULL))
    end
    for (c, mu) in penalties
        A = Vector{Float64}(mu); length(A) == M || throw(DimensionMismatch("penalties must have length M"))
        push!(keep, A); push!(tables, ToQueueTable(3, c - 1, 1, 0, pointer(A), C_NULL))
    end
    if Xref !== nothing
        XR, UR = Array{Float64,3}(Xref), Array{Float64,3}(Uref)
        (size(XR, 3) == M && size(UR, 3) == M && size(XR, 2) == size(UR, 2)) || throw(DimensionMismatch("Xref must be (n, nref, M) and Uref (m, nref, M)"))
        push!(keep, XR, UR); push!(tables, ToQueueTable(4, start, size(XR, 2), 0, pointer(XR), pointer(UR)))
    end
    status, iters, outer = Vector{Int32}(undef, M), Vector{Int32}(undef, M), Vector{Int32}(undef, M)
    cost, dJ, grad, cmax = (Vector{Float64}(undef, M) for _ in 1:4)
    X, U = Array{Float64,3}(undef, n, N, M), Array{Float64,3}(undef, m, N - 1, M)
    GC.@preserve X0 U0 XF P keep begin
        spec = Ref(ToQueueSpec(M, shared, pointer(X0), pointer(U0), XF === nothing ? C_NULL : pointer(XF), objective, constraint,
                               P === nothing ? C_NULL : pointer(P), P === nothing ? 0 : size(P, 1), 0))
        if isempty(tables)
            check(p.h, ccall((:to_solve_queue, libb200), Cint,
                             (Ptr{Cvoid}, Ref{ToQueueSpec}, Ref{ToSolveOptions}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
                              Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                             p.h, spec, o, status, iters, outer, cost, dJ, grad, cmax, X, U))
        else
            check(p.h, ccall((:to_solve_queue_tables, libb200), Cint,
                             (Ptr{Cvoid}, Ref{ToQueueSpec}, Ptr{ToQueueTable}, Int32, Ref{ToSolveOptions}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32},
                              Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}),
                             p.h, spec, tables, length(tables), o, status, iters, outer, cost, dJ, grad, cmax, X, U))
        end
    end
    (status = [SOLVE_STATUS[s + 1] for s in status], iterations = iters, iterations_outer = outer, cost = cost, dJ = dJ, gradient = grad,
     c_max = cmax, X = X, U = U)
end

# MPC plumbing: update_trajectory!(obj, Z, start) src/objective.jl:198-212 on the batched problem; Xref (n, nref), Uref (m, nref)
TO.update_trajectory!(p::BatchedProblem, Xref::Matrix{Float64}, Uref::Matrix{Float64}, start::Integer=1) =
    check(p.h, ccall((:to_update_trajectory, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Int32, Int32), p.h, Xref, Uref, size(Xref, 2), start))
# per instance: Xref (n, nref, B), Uref (m, nref, B), one start for the batch
function TO.update_trajectory!(p::BatchedProblem, Xref::Array{Float64,3}, Uref::Array{Float64,3}, start::Integer=1)
    (size(Xref, 3) == p.B && size(Uref, 3) == p.B && size(Uref, 2) == size(Xref, 2)) || throw(DimensionMismatch("Xref (n, nref, B), Uref (m, nref, B)"))
    check(p.h, ccall((:to_update_trajectories, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Int32, Int32), p.h, Xref, Uref, size(Xref, 2), start))
end
shift_trajectory!(p::BatchedProblem, steps::Integer=1) = check(p.h, ccall((:to_shift_trajectory, libb200), Cint, (Ptr{Cvoid}, Int32), p.h, steps))

# closed-loop MPC on the device (to_mpc_spec field for field): a receding-horizon simulation of every instance, no host round trip per step
struct ToMpcSpec
    nsteps::Int32; nparams::Int32
    plant_params::Ptr{Float64}; W::Ptr{Float64}; Xref::Ptr{Float64}; Uref::Ptr{Float64}
    nref::Int32; start::Int32
end
const MPC_STEPS = WeakKeyDict{BatchedProblem,Vector{Int}}()    # [steps done, nsteps] since the last mpc_setup!
# plant_params (nparams, B) or nothing; W (n_e, nsteps, B) or nothing; Xref (n, nref, B) and Uref (m, nref, B) or nothing
function mpc_setup!(p::BatchedProblem, nsteps::Integer; plant_params=nothing, W=nothing, Xref=nothing, Uref=nothing, start::Integer=1)
    P = plant_params === nothing ? nothing : Matrix{Float64}(plant_params)
    Wd = W === nothing ? nothing : Array{Float64,3}(W)
    Xr = Xref === nothing ? nothing : Array{Float64,3}(Xref)
    Ur = Uref === nothing ? nothing : Array{Float64,3}(Uref)
    P === nothing || size(P, 2) == p.B || throw(DimensionMismatch("plant_params must be (nparams, B)"))
    Wd === nothing || (size(Wd, 2) == nsteps && size(Wd, 3) == p.B) || throw(DimensionMismatch("W must be (n_e, nsteps, B)"))
    (Xr === nothing) == (Ur === nothing) || throw(ArgumentError("Xref and Uref are given together"))
    Xr === nothing || (size(Xr, 3) == p.B && size(Ur, 3) == p.B && size(Ur, 2) == size(Xr, 2)) || throw(DimensionMismatch("Xref (n, nref, B), Uref (m, nref, B)"))
    ptr(a) = a === nothing ? Ptr{Float64}(C_NULL) : pointer(a)
    GC.@preserve P Wd Xr Ur begin
        spec = ToMpcSpec(nsteps, P === nothing ? 0 : size(P, 1), ptr(P), ptr(Wd), ptr(Xr), ptr(Ur), Xr === nothing ? 0 : size(Xr, 2), start)
        check(p.h, ccall((:to_mpc_setup, libb200), Cint, (Ptr{Cvoid}, Ref{ToMpcSpec}), p.h, spec))
    end
    MPC_STEPS[p] = [0, Int(nsteps)]
    nothing
end
# enqueues `steps` MPC steps of `iterations` iLQR iterations each and returns without waiting for them
function mpc_run!(p::BatchedProblem, steps::Integer; iterations::Integer=1)
    haskey(MPC_STEPS, p) || throw(ArgumentError("mpc_run! before mpc_setup!"))
    check(p.h, ccall((:to_mpc_run, libb200), Cint, (Ptr{Cvoid}, Int32, Int32), p.h, steps, iterations))
    MPC_STEPS[p][1] += steps
    nothing
end
# (X (n, s+1, B), U (m, s, B), J (s, B)) of the s steps run since mpc_setup!
function mpc_history(p::BatchedProblem)
    haskey(MPC_STEPS, p) || throw(ArgumentError("mpc_history before mpc_setup!"))
    s = MPC_STEPS[p][1]
    n, m, _ = RD.dims(p.prob, 1)
    X = Array{Float64,3}(undef, n, s + 1, p.B); U = Array{Float64,3}(undef, m, s, p.B); J = Matrix{Float64}(undef, s, p.B)
    check(p.h, ccall((:to_mpc_history, libb200), Cint, (Ptr{Cvoid}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}), p.h, X, U, J))
    X, U, J
end
# enqueues `steps` MPC steps whose plan is solve!(p; kw...) (a budget of `iterations` iterations per step, the options solve! takes) and
# returns without waiting for them; a constrained problem gets per-instance penalties first, so each instance takes its own outer steps
function mpc_solve!(p::BatchedProblem, steps::Integer; kw...)
    haskey(MPC_STEPS, p) || throw(ArgumentError("mpc_solve! before mpc_setup!"))
    o = solve_options(kw)
    check(p.h, ccall((:to_mpc_solve, libb200), Cint, (Ptr{Cvoid}, Int32, Ref{ToSolveOptions}), p.h, steps, o))
    MPC_STEPS[p][1] += steps
    nothing
end
# the solve statistics of the s steps run since mpc_setup!, (s, B) each; a step mpc_run! took holds status -1 (:NOT_SOLVED here), iterations 0,
# iterations_outer 0, c_max NaN
function mpc_solve_history(p::BatchedProblem)
    haskey(MPC_STEPS, p) || throw(ArgumentError("mpc_solve_history before mpc_setup!"))
    s = MPC_STEPS[p][1]
    status, iters, outer = (Matrix{Int32}(undef, s, p.B) for _ in 1:3)
    cmax = Matrix{Float64}(undef, s, p.B)
    check(p.h, ccall((:to_mpc_solve_history, libb200), Cint, (Ptr{Cvoid}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}, Ptr{Float64}),
                     p.h, status, iters, outer, cmax))
    (status = [st < 0 ? :NOT_SOLVED : SOLVE_STATUS[st + 1] for st in status], iterations = iters, iterations_outer = outer, c_max = cmax)
end

# multi-GPU (one process per GPU, e.g. under MPI.jl + NCCL.jl): the only collective is the {sum J, max violation} all-reduce.
# `to_reduce_merit_async` queues the per-GPU reduction behind the iteration in flight and makes `stream` (the CUDA.jl
# stream the NCCL call is issued on) wait for it; `merit_device_ptr` is the 2-double buffer to all-reduce in place.
reduce_merit_async!(p::BatchedProblem, stream::Ptr{Cvoid}) = check(p.h, ccall((:to_reduce_merit_async, libb200), Cint, (Ptr{Cvoid}, Ptr{Cvoid}), p.h, stream))
function merit_device_ptr(p::BatchedProblem)
    r = Ref{Ptr{Cvoid}}(C_NULL)
    check(p.h, ccall((:to_merit_device_ptr, libb200), Cint, (Ptr{Cvoid}, Ref{Ptr{Cvoid}}), p.h, r)); r[]
end

end # module
