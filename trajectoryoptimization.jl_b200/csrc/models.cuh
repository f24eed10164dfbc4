// models.cuh -- device dynamics of the models on the hot path, templated over the scalar type so the same
// text runs with `double` (rollout) and with in-register forward-mode dual numbers (dynamics Jacobians).
//
// What each model mirrors (reference file:line under /root/reference):
//   Cartpole          docs/src/model.md:32-51            (mc, mp, l, g at :27)
//   Quadrotor         examples/Quadrotor.ipynb cell 8 forces/moments + cell 4 parameters; rigid-body
//                     kinematics from RobotDynamics.jl `RigidBody` (world-frame velocity, scalar-first quaternion)
//   DoubleIntegrator  examples/quickstart.jl:15-20
//   Acrobot           RobotZoo.jl `Acrobot` (not present in the reference tree)
// Discretisation: RobotDynamics.jl's explicit rules with zero-order hold (explicit_step): Euler, RK2, RK3 or RK4, the
// integrator `Problem` selects (src/problem.jl:119-123; RK4 by default) and `rollout!` steps through (src/problem.jl:334-340).
#pragma once
#include "common.cuh"

// ---------------------------------------------------------------------------------------------------
// Dual number with P partials kept in registers (ForwardDiff.Dual analogue).
template <int P>
struct Dual {
    double v;
    double d[P];
    __device__ __forceinline__ Dual() {}
    __device__ __forceinline__ Dual(double a) : v(a) {
#pragma unroll
        for (int i = 0; i < P; i++) d[i] = 0.0;
    }
};
#define DUAL_BIN template <int P> __device__ __forceinline__ Dual<P>
DUAL_BIN operator+(const Dual<P>& a, const Dual<P>& b) { Dual<P> r; r.v = a.v + b.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = a.d[i] + b.d[i]; return r; }
DUAL_BIN operator-(const Dual<P>& a, const Dual<P>& b) { Dual<P> r; r.v = a.v - b.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = a.d[i] - b.d[i]; return r; }
DUAL_BIN operator-(const Dual<P>& a) { Dual<P> r; r.v = -a.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = -a.d[i]; return r; }
DUAL_BIN operator*(const Dual<P>& a, const Dual<P>& b) { Dual<P> r; r.v = a.v * b.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = fma(a.d[i], b.v, a.v * b.d[i]); return r; }
DUAL_BIN operator/(const Dual<P>& a, const Dual<P>& b) { Dual<P> r; double inv = 1.0 / b.v; r.v = a.v * inv;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv; return r; }
DUAL_BIN operator+(const Dual<P>& a, double b) { Dual<P> r = a; r.v += b; return r; }
DUAL_BIN operator+(double b, const Dual<P>& a) { Dual<P> r = a; r.v += b; return r; }
DUAL_BIN operator-(const Dual<P>& a, double b) { Dual<P> r = a; r.v -= b; return r; }
DUAL_BIN operator-(double b, const Dual<P>& a) { Dual<P> r = -a; r.v += b; return r; }
DUAL_BIN operator*(const Dual<P>& a, double b) { Dual<P> r; r.v = a.v * b;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = a.d[i] * b; return r; }
DUAL_BIN operator*(double b, const Dual<P>& a) { return a * b; }
DUAL_BIN operator/(const Dual<P>& a, double b) { return a * (1.0 / b); }
DUAL_BIN dsin(const Dual<P>& a) { Dual<P> r; double s, c; sincos(a.v, &s, &c); r.v = s;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = c * a.d[i]; return r; }
DUAL_BIN dcos(const Dual<P>& a) { Dual<P> r; double s, c; sincos(a.v, &s, &c); r.v = c;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = -s * a.d[i]; return r; }
// max(0,x): derivative 0 on a tie (the constant is returned), 1 for x > 0  -- SURVEY.md section 7
DUAL_BIN drelu(const Dual<P>& a) { return a.v > 0 ? a : Dual<P>(0.0); }
__device__ __forceinline__ double dsin(double a) { return sin(a); }
__device__ __forceinline__ double dcos(double a) { return cos(a); }
__device__ __forceinline__ double drelu(double a) { return a > 0 ? a : 0.0; }
template <class S> __device__ __forceinline__ S lift(double a) { return S(a); }
// the remaining operations of the recorded-program interpreter (include/trajopt_b200.h to_expr_op), value + P partials
DUAL_BIN dexp(const Dual<P>& a) { Dual<P> r; r.v = exp(a.v);
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = r.v * a.d[i]; return r; }
DUAL_BIN dlog(const Dual<P>& a) { Dual<P> r; r.v = log(a.v); const double iv = 1.0 / a.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = iv * a.d[i]; return r; }
DUAL_BIN dsqrt(const Dual<P>& a) { Dual<P> r; r.v = sqrt(a.v); const double f = 0.5 / r.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = f * a.d[i]; return r; }
DUAL_BIN dtanh(const Dual<P>& a) { Dual<P> r; r.v = tanh(a.v); const double f = 1.0 - r.v * r.v;
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = f * a.d[i]; return r; }
DUAL_BIN dpowc(const Dual<P>& a, double e) { Dual<P> r; r.v = pow(a.v, e); const double f = e * pow(a.v, e - 1.0);
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = f * a.d[i]; return r; }
__device__ __forceinline__ double dexp(double a) { return exp(a); }
__device__ __forceinline__ double dlog(double a) { return log(a); }
__device__ __forceinline__ double dsqrt(double a) { return sqrt(a); }
__device__ __forceinline__ double dtanh(double a) { return tanh(a); }
__device__ __forceinline__ double dpowc(double a, double e) { return pow(a, e); }

// ---------------------------------------------------------------------------------------------------
template <int MODEL> struct ModelDims;
template <> struct ModelDims<MODEL_CARTPOLE> { static constexpr int n = 4, m = 1; };
template <> struct ModelDims<MODEL_QUADROTOR> { static constexpr int n = 13, m = 4; };
template <> struct ModelDims<MODEL_ACROBOT> { static constexpr int n = 4, m = 1; };
// the double integrator comes in two sizes (BASELINE.json configs[0] 1-D, examples/quickstart.jl 2-D)
constexpr int MODEL_DOUBLE_INTEGRATOR_2D = 16;
template <> struct ModelDims<MODEL_DOUBLE_INTEGRATOR> { static constexpr int n = 2, m = 1; };
template <> struct ModelDims<MODEL_DOUBLE_INTEGRATOR_2D> { static constexpr int n = 4, m = 2; };
// user dynamics recorded as programs (TO_MODEL_EXPR), single or hybrid / variable-dimension models: instantiated for three padded size
// classes, (4, 2) -- the reference's hybrid example (test/hybrid_dynamics_model.jl:15-54) --, (8, 4) and (16, 8).  A problem runs on the
// smallest class that holds its largest per-knot dimensions (capi.cu to_recorded_dims); the padded m (2, 4 or 8) names the class.
constexpr int MODEL_EXPR_42 = 20, MODEL_EXPR_84 = 21, MODEL_EXPR_168 = 22;
template <> struct ModelDims<MODEL_EXPR_42> { static constexpr int n = 4, m = 2; };
template <> struct ModelDims<MODEL_EXPR_84> { static constexpr int n = 8, m = 4; };
template <> struct ModelDims<MODEL_EXPR_168> { static constexpr int n = 16, m = 8; };
template <int MODEL> constexpr bool is_recorded = MODEL == MODEL_EXPR_42 || MODEL == MODEL_EXPR_84 || MODEL == MODEL_EXPR_168;

// a b - c c (the Cartpole's mass-matrix determinant).  With dual numbers the value is written as the one rounding fma(a, b, -(c c)): the
// compiler is free to contract either product, and it chose differently when the parameters came from shared memory (per-instance
// parameters) than from the parameter bank; this is the form the shared kernels have always computed.
// With doubles the shared kernels differ among themselves: the generic line search (rollout_generic) computes fma(a, b, -(c c)), and its
// per-instance variant contracted c c instead (one ulp off in the merit).  DET_FMA writes that kernel's form out; every other instantiation
// keeps the plain expression, and so the code it has always compiled to (writing fma everywhere changes the shared rollout and the fast
// line-search kernels).
template <bool DET_FMA>
__device__ __forceinline__ double det_sub_square(double a, double b, double c) {
    if constexpr (DET_FMA) return fma(a, b, -(c * c));
    else return a * b - c * c;
}
template <bool DET_FMA, int P>
__device__ __forceinline__ Dual<P> det_sub_square(const Dual<P>& a, const Dual<P>& b, const Dual<P>& c) {
    const Dual<P> ab = a * b, cc = c * c;
    Dual<P> r;
    r.v = fma(a.v, b.v, -cc.v);
#pragma unroll
    for (int i = 0; i < P; i++) r.d[i] = ab.d[i] - cc.d[i];
    return r;
}

template <int MODEL, class S, bool DET_FMA = false>
__device__ __forceinline__ void dynamics(const double* __restrict__ p, const S* x, const S* u, S* xd) {
    if constexpr (is_recorded<MODEL>) {
        // `p` is the knot's DevDyn (model_params): interpret the recorded program with the scalar type S (double or dual numbers); the
        // outputs are the last n_out instructions, the unused state slots of the next knot stay zero
        constexpr int n = ModelDims<MODEL>::n;
        const DevDyn& dy = *reinterpret_cast<const DevDyn*>(p);
        S reg[TO_EXPR_LEN];
        for (int i = 0; i < dy.prog_len; i++) {
            const int op = dy.prog[3 * i], a = dy.prog[3 * i + 1], b = dy.prog[3 * i + 2];
            S r = lift<S>(0.0);
            switch (op) {
                case 0: r = lift<S>(dy.pconst[a]); break;
                case 1: r = x[a]; break;
                case 2: r = u[a]; break;
                case 3: r = reg[a] + reg[b]; break;
                case 4: r = reg[a] - reg[b]; break;
                case 5: r = reg[a] * reg[b]; break;
                case 6: r = reg[a] / reg[b]; break;
                case 7: r = -reg[a]; break;
                case 8: r = dsin(reg[a]); break;
                case 9: r = dcos(reg[a]); break;
                case 10: r = dexp(reg[a]); break;
                case 11: r = dlog(reg[a]); break;
                case 12: r = dsqrt(reg[a]); break;
                case 13: r = dpowc(reg[a], dy.pconst[b]); break;
                case 14: r = dtanh(reg[a]); break;
                case 15: r = reg[a] + dy.pconst[b]; break;
                case 16: r = reg[a] * dy.pconst[b]; break;
                case 17: r = reg[a] * (1.0 / dy.pconst[b]); break;
                case 18: r = lift<S>(dy.pconst[b]) / reg[a]; break;
                case 19: r = dy.pconst[b] - reg[a]; break;
            }
            reg[i] = r;
        }
#pragma unroll
        for (int i = 0; i < n; i++) xd[i] = (i < dy.n_out) ? reg[dy.prog_len - dy.n_out + i] : lift<S>(0.0);
    } else if constexpr (MODEL == MODEL_DOUBLE_INTEGRATOR || MODEL == MODEL_DOUBLE_INTEGRATOR_2D) {
        constexpr int dim = ModelDims<MODEL>::m;
        const double inv_mass = p[1];   // 1/mass, precomputed on the host
#pragma unroll
        for (int i = 0; i < dim; i++) { xd[i] = x[dim + i]; xd[dim + i] = u[i] * inv_mass; }
    } else if constexpr (MODEL == MODEL_CARTPOLE) {
        const double mc = p[0], mp = p[1], l = p[2], g = p[3];
        S s = dsin(x[1]), c = dcos(x[1]);
        S qd1 = x[2], qd2 = x[3];
        S h11 = lift<S>(mc + mp), h12 = (mp * l) * c, h22 = lift<S>(mp * l * l);
        S r1 = (-mp * l) * (qd2 * s) * qd2 - u[0];
        S r2 = (mp * g * l) * s;
        S idet = lift<S>(1.0) / det_sub_square<DET_FMA>(h11, h22, h12);
        xd[0] = qd1; xd[1] = qd2;
        xd[2] = -(h22 * r1 - h12 * r2) * idet;
        xd[3] = -(h11 * r2 - h12 * r1) * idet;
    } else if constexpr (MODEL == MODEL_QUADROTOR) {
        const double mass = p[0], J1 = p[1], J2 = p[2], J3 = p[3];
        const double gx = p[4], gy = p[5], gz = p[6], L = p[7], kf = p[8], km = p[9];
        const double inv_mass = p[10], iJ1 = p[11], iJ2 = p[12], iJ3 = p[13];   // reciprocals precomputed on the host (to_create)
        S qw = x[3], qx = x[4], qy = x[5], qz = x[6];
        S wx = x[10], wy = x[11], wz = x[12];
        S F1 = drelu(kf * u[0]), F2 = drelu(kf * u[1]), F3 = drelu(kf * u[2]), F4 = drelu(kf * u[3]);
        S Fz = F1 + F2 + F3 + F4;
        // world force = m g + q * [0,0,Fz]  with  q*r = (w^2 - v'v) r + 2 v (v'r) + 2 w (v x r)
        S vv = qx * qx + qy * qy + qz * qz;
        S ww = qw * qw - vv;
        S vr = qz * Fz;
        S Fwx = 2.0 * (qx * vr) + 2.0 * (qw * (qy * Fz));
        S Fwy = 2.0 * (qy * vr) - 2.0 * (qw * (qx * Fz));
        S Fwz = ww * Fz + 2.0 * (qz * vr);
        S M1 = km * u[0], M2 = km * u[1], M3 = km * u[2], M4 = km * u[3];
        S t1 = L * (F2 - F4), t2 = L * (F3 - F1), t3 = (M1 - M2 + M3 - M4);
        xd[0] = x[7]; xd[1] = x[8]; xd[2] = x[9];
        xd[3] = -0.5 * (qx * wx + qy * wy + qz * wz);
        xd[4] = 0.5 * (qw * wx + qy * wz - qz * wy);
        xd[5] = 0.5 * (qw * wy + qz * wx - qx * wz);
        xd[6] = 0.5 * (qw * wz + qx * wy - qy * wx);
        xd[7] = (mass * gx + Fwx) * inv_mass;
        xd[8] = (mass * gy + Fwy) * inv_mass;
        xd[9] = (mass * gz + Fwz) * inv_mass;
        S Jw1 = J1 * wx, Jw2 = J2 * wy, Jw3 = J3 * wz;
        xd[10] = (t1 - (wy * Jw3 - wz * Jw2)) * iJ1;
        xd[11] = (t2 - (wz * Jw1 - wx * Jw3)) * iJ2;
        xd[12] = (t3 - (wx * Jw2 - wy * Jw1)) * iJ3;
    } else if constexpr (MODEL == MODEL_ACROBOT) {
        const double l1 = p[0], l2 = p[1], m1 = p[2], m2 = p[3], J1 = p[4], J2 = p[5], fr = p[6], g = p[7];
        S th1 = x[0], th2 = x[1], th1d = x[2], th2d = x[3];
        S c1 = dcos(th1), s2 = dsin(th2), c2 = dcos(th2), c12 = dcos(th1 + th2);
        S m11 = (m1 * l1 * l1 + J1 + J2) + m2 * ((l1 * l1 + l2 * l2) + (2.0 * l1 * l2) * c2);
        S m12 = m2 * ((l2 * l2 + J2) + (l1 * l2) * c2);
        S m22 = lift<S>(l2 * l2 * m2 + J2);
        S tmp = (l1 * l2 * m2) * s2;
        S b1 = -(2.0 * (th1d * th2d) + th2d * th2d) * tmp;
        S b2 = tmp * (th1d * th1d);
        S f1 = fr * th1d, f2 = fr * th2d;
        S g1 = (((m1 + m2) * l2) * c1 + (m2 * l2) * c12) * g;
        S g2 = (m2 * l2 * g) * c12;
        S r1 = -b1 - g1 - f1;
        S r2 = u[0] - b2 - g2 - f2;
        S idet = lift<S>(1.0) / (m11 * m22 - m12 * m12);
        xd[0] = th1d; xd[1] = th2d;
        xd[2] = (m22 * r1 - m12 * r2) * idet;
        xd[3] = (m11 * r2 - m12 * r1) * idet;
    }
}

// One step of the explicit rule RULE (include/trajopt_b200.h to_integration), zero-order hold on u, each k_i scaled by h as RobotDynamics
// does before it is used:
//   1 Euler  x+ = x + k1
//   2 RK2    (explicit midpoint) k2 = h f(x + k1/2);  x+ = x + k2
//   3 RK3    (Kutta) k2 = h f(x + k1/2);  k3 = h f(x - k1 + 2 k2);  x+ = x + (k1 + 4 k2 + k3)/6
//   4 RK4    x+ = x + (k1 + 2k2 + 2k3 + k4)/6
// with k1 = h f(x, u).  Every rule reads x_i for the last time where it writes xn_i, so xn may be x (rollout_compact steps in place).
// The weights of every rule sum to one, which keeps the closed-form position / velocity Jacobian columns exact (rollout.cu SeedList).
// The 1/6 of RK3 and RK4 is a product, as RK4 has always computed it: an FP64 division is a multi-instruction sequence on the line search's
// dependency chain (RK3 written with / 6, as the oracle writes it, took the BASELINE line search's pass 1 to 0.49 ms, against 0.29 ms as a product).
// DET_FMA: the Cartpole's determinant as one explicit fma (det_sub_square)
template <int MODEL, class S, int RULE, bool DET_FMA = false>
__device__ __forceinline__ void explicit_step(const double* __restrict__ p, const S* x, const S* u, double h, S* xn) {
    static_assert(RULE >= 1 && RULE <= 4, "to_integration: TO_EULER .. TO_RK4");
    constexpr int n = ModelDims<MODEL>::n;
    if constexpr (is_recorded<MODEL>) {     // a discrete jump map is applied as is
        if (reinterpret_cast<const DevDyn*>(p)->discrete) { dynamics<MODEL, S>(p, x, u, xn); return; }
    }
    if constexpr (RULE == 1) {
        S k[n];
        dynamics<MODEL, S, DET_FMA>(p, x, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) xn[i] = x[i] + k[i] * h;
    } else if constexpr (RULE == 2) {
        S k[n], xt[n];
        dynamics<MODEL, S, DET_FMA>(p, x, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; xt[i] = x[i] + k[i] * 0.5; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) xn[i] = x[i] + k[i] * h;
    } else if constexpr (RULE == 3) {
        S k1[n], k[n], xt[n];                   // k1 becomes k1 + 4 k2 once the third stage's point is formed
        dynamics<MODEL, S, DET_FMA>(p, x, u, k1);
#pragma unroll
        for (int i = 0; i < n; i++) { k1[i] = k1[i] * h; xt[i] = x[i] + k1[i] * 0.5; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; xt[i] = x[i] - k1[i] + 2.0 * k[i]; k1[i] = k1[i] + 4.0 * k[i]; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; xn[i] = x[i] + (k1[i] + k[i]) * (1.0 / 6.0); }
    } else {
        S k[n], acc[n], xt[n];
        dynamics<MODEL, S, DET_FMA>(p, x, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; acc[i] = k[i]; xt[i] = x[i] + k[i] * 0.5; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; acc[i] = acc[i] + 2.0 * k[i]; xt[i] = x[i] + k[i] * 0.5; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; acc[i] = acc[i] + 2.0 * k[i]; xt[i] = x[i] + k[i]; }
        dynamics<MODEL, S, DET_FMA>(p, xt, u, k);
#pragma unroll
        for (int i = 0; i < n; i++) { k[i] = k[i] * h; xn[i] = x[i] + (acc[i] + k[i]) * (1.0 / 6.0); }
    }
}

// dispatch a templated launcher on the runtime model id / dimension
#define TO_DISPATCH_MODEL(model_id, m_dim, CALL)                                                   \
    switch (model_id) {                                                                            \
        case MODEL_DOUBLE_INTEGRATOR:                                                              \
            if ((m_dim) == 1) { constexpr int MODEL = MODEL_DOUBLE_INTEGRATOR; CALL; }             \
            else { constexpr int MODEL = MODEL_DOUBLE_INTEGRATOR_2D; CALL; }                       \
            break;                                                                                 \
        case MODEL_CARTPOLE: { constexpr int MODEL = MODEL_CARTPOLE; CALL; } break;                \
        case MODEL_QUADROTOR: { constexpr int MODEL = MODEL_QUADROTOR; CALL; } break;              \
        case MODEL_ACROBOT: { constexpr int MODEL = MODEL_ACROBOT; CALL; } break;                  \
        case MODEL_EXPR:                                                                           \
            if ((m_dim) == 2) { constexpr int MODEL = MODEL_EXPR_42; CALL; }                       \
            else if ((m_dim) == 4) { constexpr int MODEL = MODEL_EXPR_84; CALL; }                  \
            else { constexpr int MODEL = MODEL_EXPR_168; CALL; }                                   \
            break;                                                                                 \
    }

// dispatch on the problem's explicit rule (DevProblem::integration): RULE = RULE_EULER .. RULE_RK4
#define TO_DISPATCH_RULE(rule, CALL)                                                               \
    switch (rule) {                                                                                \
        case RULE_EULER: { constexpr int RULE = RULE_EULER; CALL; } break;                         \
        case RULE_RK2: { constexpr int RULE = RULE_RK2; CALL; } break;                             \
        case RULE_RK3: { constexpr int RULE = RULE_RK3; CALL; } break;                             \
        default: { constexpr int RULE = RULE_RK4; CALL; } break;                                   \
    }

// what explicit_step / dynamics take as `p` at knot k: the shared parameter vector (INST = false); INST: `row`, the copy of instance b's parameters
// the kernel made with stage_model_params; recorded programs: the DevDyn of knot k (their constants are never per instance)
template <int MODEL, bool INST = false>
__device__ __forceinline__ const double* model_params(const DevProblem& P, const double* row, int k) {
    if constexpr (is_recorded<MODEL>) return reinterpret_cast<const double*>(&P.dyn[P.dyn_index[k]]);
    else if constexpr (INST) return row;
    else return P.params;
}
// row[0 .. TO_NPARAM) = the parameters of instance b (common.cuh model_param), `row` in shared memory: read from there, the dynamics compile
// to the same FP64 operations as with the shared vector in the parameter bank (a copy in registers loses FMA contractions)
template <bool INST>
__device__ __forceinline__ void stage_model_params(const DevProblem& P, int b, double* row) {
#pragma unroll
    for (int i = 0; i < TO_NPARAM; i++) row[i] = model_param<INST>(P, b, i);
}
