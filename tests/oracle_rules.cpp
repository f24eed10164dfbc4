// oracle_rules.cpp -- the CPU oracle (oracle/) with every explicit rule of include/trajopt_b200.h to_integration.
//
// The oracle steps with RK4 or RK3 (oracle/models.hpp rk4_step, orc_set_integrator).  This translation unit compiles the oracle's own sources
// unchanged and puts one step in front of theirs: Euler and RK2 in the operation order of csrc/models.cuh explicit_step, every other case
// (RK4, RK3, a jump map) handed to the oracle's step.  It exports orc_set_integration / orc_get_integration, so that a problem opened on this
// library takes Problem(..., integration) through the same call as the device (tests/integration_rules.py RulesOracleProblem).  Test
// infrastructure: built by tests/integration_rules.py into tests/_build/liboracle_rules.so (git-ignored).
#define rk4_step oracle_step
#include "../oracle/models.hpp"
#undef rk4_step

namespace oracle {
// RobotDynamics' explicit rules with zero-order hold, each k_i scaled by h before it is used:
//   1 Euler  x+ = x + h f(x, u);   2 RK2 (explicit midpoint)  k1 = h f(x, u); x+ = x + h f(x + k1/2, u)
template <class S>
inline void rk4_step(const ModelParams& mp, const S* x, const S* u, double h, S* xn) {
    const bool jump = mp.id == MODEL_EXPR && mp.prog->discrete;          // a jump map is applied as it is
    if (jump || (mp.integrator != 1 && mp.integrator != 2)) { oracle_step<S>(mp, x, u, h, xn); return; }
    const int n = mp.n;
    S k[MAXN], xt[MAXN];
    dynamics<S>(mp, x, u, k);
    if (mp.integrator == 1) {
        for (int i = 0; i < n; i++) xn[i] = x[i] + k[i] * h;
        return;
    }
    for (int i = 0; i < n; i++) { k[i] = k[i] * h; xt[i] = x[i] + k[i] * 0.5; }
    dynamics<S>(mp, xt, u, k);
    for (int i = 0; i < n; i++) xn[i] = x[i] + k[i] * h;
}
}  // namespace oracle

#include "../oracle/oracle_capi.cpp"

extern "C" {
// to_set_integration / to_get_integration: 1 Euler, 2 RK2, 3 RK3, 4 RK4
int orc_set_integration(orc_handle* h, int32_t rule) {
    if (rule < 1 || rule > 4) return fail(h, TO_EINVAL, "orc_set_integration: unknown integration rule " + std::to_string(rule));
    h->P.model.integrator = rule;
    h->P.J_valid = false;
    return TO_OK;
}
int orc_get_integration(orc_handle* h, int32_t* rule) {
    *rule = h->P.model.integrator;
    return TO_OK;
}
}
