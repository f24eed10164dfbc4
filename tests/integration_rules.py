"""NumPy restatements of the explicit rules of include/trajopt_b200.h to_integration (RobotDynamics' Euler, RK2, RK3, RK4 with zero-order
hold on u, each k_i scaled by h before it is used), and the oracle with every rule.

``RulesOracleProblem`` is an ``OracleProblem`` opened on tests/oracle_rules.cpp, the oracle's own sources with Euler and RK2 added and
``orc_set_integration`` / ``orc_get_integration`` exported, so ``Problem(..., integration)`` reaches it through OracleProblem's ``_raw_call``
as it reaches the device.  Shared by tests/test_integration_args.py (CPU) and tests/test_gpu_integration.py.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import trajopt_b200 as TO
from oracle_binding import ORACLE_DIR, ROOT, OracleProblem, oracle_dynamics

HERE = os.path.dirname(os.path.abspath(__file__))
RULES_SRC = os.path.join(HERE, "oracle_rules.cpp")
RULES_LIB = os.path.join(HERE, "_build", "liboracle_rules.so")
_rules_lib = None


def build_rules_oracle():
    """tests/_build/liboracle_rules.so, rebuilt when it is older than its source or the oracle's (the flags of oracle/Makefile)"""
    srcs = [RULES_SRC, os.path.join(ROOT, "include", "trajopt_b200.h")] + [os.path.join(ORACLE_DIR, f) for f in ("oracle.hpp", "models.hpp", "oracle_capi.cpp")]
    if not os.path.exists(RULES_LIB) or any(os.path.getmtime(f) > os.path.getmtime(RULES_LIB) for f in srcs):
        os.makedirs(os.path.dirname(RULES_LIB), exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        subprocess.check_call([cxx, "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-variable",
                               "-Wno-maybe-uninitialized", "-shared", "-o", RULES_LIB, RULES_SRC])
    return RULES_LIB


def load_rules_oracle():
    global _rules_lib
    if _rules_lib is None:
        _rules_lib = C.CDLL(build_rules_oracle())
        _rules_lib.orc_last_error.restype = C.c_char_p
        _rules_lib.orc_last_error.argtypes = [C.c_void_p]
    return _rules_lib


class RulesOracleProblem(OracleProblem):
    """an OracleProblem on the oracle with every explicit rule"""

    def _open(self):
        self._lib = load_rules_oracle()
        self._h = C.c_void_p()
        rc = self._lib.orc_create(C.byref(self.spec.c), C.byref(self._h))
        if rc:
            msg = self._lib.orc_last_error(None).decode()
            raise {TO.capi.TO_EDIM: TO.DimensionMismatch, TO.capi.TO_EINVAL: TO.ArgumentError}.get(rc, TO.TrajOptError)(msg)


RULES = {"Euler": TO.Euler, "RK2": TO.RK2, "RK3": TO.RK3, "RK4": TO.RK4}


def step(f, x, u, h, rule):
    """x+ of one step of `rule` (a name of RULES) with the continuous dynamics f(x, u), in the operation order of csrc/models.cuh"""
    k1 = f(x, u) * h
    if rule == "Euler":
        return x + k1
    k2 = f(x + k1 * 0.5, u) * h
    if rule == "RK2":
        return x + k2
    if rule == "RK3":
        k3 = f(x - k1 + 2.0 * k2, u) * h
        return x + ((k1 + 4.0 * k2) + k3) * (1.0 / 6.0)
    k3 = f(x + k2 * 0.5, u) * h
    k4 = f(x + k3, u) * h
    return x + ((k1 + 2.0 * k2) + 2.0 * k3 + k4) * (1.0 / 6.0)


def model_step(model, rule):
    """(x, u, h) -> x+ for a built-in model, on the oracle's continuous dynamics"""
    return lambda x, u, h: step(lambda a, b: oracle_dynamics(model, a, b), np.asarray(x, float), np.asarray(u, float), h, rule)


def rollout(stepper, x0, U, dt):
    """X[N, n] from x0 under the controls U[N-1, m] and the steps dt[N-1]"""
    X = np.empty((len(U) + 1, len(x0)))
    X[0] = x0
    for k in range(len(U)):
        X[k + 1] = stepper(X[k], U[k], dt[k])
    return X


def jacobian_fd(stepper, x, u, h, eps=1e-6):
    """[A B] = d x+ / d [x; u] by central differences, n x (n + m)"""
    n, m = len(x), len(u)
    J = np.empty((n, n + m))
    for j in range(n + m):
        e = np.zeros(n + m)
        e[j] = eps * max(1.0, abs(np.concatenate([x, u])[j]))
        xp, up = x + e[:n], u + e[n:]
        xm, um = x - e[:n], u - e[n:]
        J[:, j] = (stepper(xp, up, h) - stepper(xm, um, h)) / (2.0 * e[j])
    return J


def double_integrator_step_errors(X, U, h, mass):
    """(position, velocity) of x_k+1 minus the exact step of x'' = u / mass from x_k under a constant u_k, for every knot: [N-1, dim] each"""
    dim = U.shape[-1]
    a = U / mass
    r, v = X[:-1, :dim], X[:-1, dim:]
    return X[1:, :dim] - (r + h[:, None] * v + 0.5 * (h * h)[:, None] * a), X[1:, dim:] - (v + h[:, None] * a)
