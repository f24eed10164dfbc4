// oracle_classes.cpp -- the CPU oracle (oracle/) with every explicit rule (tests/oracle_rules.cpp) and the padded size classes (4, 2),
// (8, 4) and (16, 8) of recorded-program problems (include/trajopt_b200.h to_recorded_dims).
//
// The oracle interprets recorded programs at any n <= MAXN, m <= MAXM, but its orc_create takes them on the padded layout (4, 2) only
// (oracle/models.hpp default_model).  This translation unit compiles the oracle's own sources unchanged and puts two things in front of
// them: an orc_create that derives the problem's size class from to_spec.nx / nu with the rule of to_recorded_dims, refuses any other
// to_spec.n, m with to_create's messages, and hands the spec to the oracle's orc_create; and a default_model that gives recorded programs
// that class.  It exports orc_recorded_dims, the rule stated on the oracle's side.  Test infrastructure: built by
// tests/recorded_classes.py into tests/_build/liboracle_classes.so (git-ignored).
#include <algorithm>
#include <string>

#define default_model oracle_default_model
#define rk4_step oracle_step
#include "../oracle/models.hpp"
#undef rk4_step
#undef default_model

namespace oracle {
// the class of the spec orc_create is opening (set by orc_create below before it calls the oracle's)
static int g_class_n = 4, g_class_m = 2;
inline ModelParams default_model(int id, int dim = 1) {
    ModelParams mp = oracle_default_model(id, dim);
    if (id == MODEL_EXPR) { mp.n = g_class_n; mp.m = g_class_m; }
    return mp;
}
// the smallest of (4, 2), (8, 4), (16, 8) that holds nx_max states and nu_max controls; false past (16, 8)
inline bool recorded_dims(int nx_max, int nu_max, int& n, int& m) {
    for (int s = 4; s <= 16; s *= 2)
        if (nx_max <= s && nu_max <= s / 2) { n = s; m = s / 2; return true; }
    return false;
}
}  // namespace oracle

#define orc_create oracle_create
#include "oracle_rules.cpp"
#undef orc_create

extern "C" {
int orc_recorded_dims(int32_t nx_max, int32_t nu_max, int32_t* n, int32_t* m) {
    if (!n || !m || nx_max < 1 || nu_max < 0) return TO_EINVAL;
    int a = 0, b = 0;
    if (!recorded_dims(nx_max, nu_max, a, b)) return TO_EDIM;
    *n = a; *m = b;
    return TO_OK;
}

int orc_create(const to_spec* s, orc_handle** out) {
    if (s && out && s->model == MODEL_EXPR) {
        *out = nullptr;
        if (s->N < 2 || !s->nx || !s->nu) return fail(nullptr, TO_EINVAL, "recorded-program models: null dyn / dyn_index / nx / nu");
        int nx_max = 0, nu_max = 0;
        for (int k = 0; k < s->N; k++) {
            if (s->nx[k] < 1 || s->nu[k] < 0) return fail(nullptr, TO_EINVAL, "recorded-program models: a knot has fewer than 1 state or 0 controls");
            nx_max = std::max(nx_max, (int)s->nx[k]); nu_max = std::max(nu_max, (int)s->nu[k]);
        }
        int n = 0, m = 0;
        if (!recorded_dims(nx_max, nu_max, n, m))
            return fail(nullptr, TO_EDIM, "recorded-program models: at most 16 states and 8 controls per knot, the largest has (" + std::to_string(nx_max) + ", " +
                        std::to_string(nu_max) + ")");
        if (s->n != n || s->m != m)
            return fail(nullptr, TO_EDIM, "recorded-program models: largest per-knot dimensions (" + std::to_string(nx_max) + ", " + std::to_string(nu_max) +
                        ") run on the padded size class n = " + std::to_string(n) + ", m = " + std::to_string(m) + " (to_recorded_dims), not n = " +
                        std::to_string(s->n) + ", m = " + std::to_string(s->m));
        g_class_n = n; g_class_m = m;
    }
    return oracle_create(s, out);
}
}
