"""User dynamics models of the padded size classes (8, 4) and (16, 8) (csrc/models.cuh MODEL_EXPR_84 / MODEL_EXPR_168), shared by the CPU
and GPU tests of those classes: programs that between them record every op code in each class, a recorded copy of the Quadrotor, a planar
quadrotor, a 7-joint arm, the closed form of the padded rows and columns of [A B], and ``ClassesOracleProblem``, an ``OracleProblem`` opened
on tests/oracle_classes.cpp: the oracle's own sources with every explicit rule and the size classes, which the oracle's orc_create does not
take (it opens recorded programs on the (4, 2) layout only)."""
import ctypes as C
import os
import subprocess

import numpy as np

import trajopt_b200 as TO
from dynamics_programs import constant_rate, powers, transcendental
from oracle_binding import ORACLE_DIR, ROOT, OracleProblem

K = TO.capi
HERE = os.path.dirname(os.path.abspath(__file__))
CLASSES_SRC = os.path.join(HERE, "oracle_classes.cpp")
CLASSES_LIB = os.path.join(HERE, "_build", "liboracle_classes.so")
_classes_lib = None


def build_classes_oracle():
    """tests/_build/liboracle_classes.so, rebuilt when it is older than its sources (the flags of oracle/Makefile)"""
    srcs = [CLASSES_SRC, os.path.join(HERE, "oracle_rules.cpp"), os.path.join(ROOT, "include", "trajopt_b200.h")] + \
        [os.path.join(ORACLE_DIR, f) for f in ("oracle.hpp", "models.hpp", "oracle_capi.cpp")]
    if not os.path.exists(CLASSES_LIB) or any(os.path.getmtime(f) > os.path.getmtime(CLASSES_LIB) for f in srcs):
        os.makedirs(os.path.dirname(CLASSES_LIB), exist_ok=True)
        cxx = "/usr/bin/g++" if os.access("/usr/bin/g++", os.X_OK) else "g++"
        tmp = f"{CLASSES_LIB}.{os.getpid()}"
        subprocess.check_call([cxx, "-O3", "-march=x86-64-v3", "-fopenmp", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-variable",
                               "-Wno-maybe-uninitialized", "-shared", "-o", tmp, CLASSES_SRC])
        os.replace(tmp, CLASSES_LIB)
    return CLASSES_LIB


def load_classes_oracle():
    global _classes_lib
    if _classes_lib is None:
        _classes_lib = C.CDLL(build_classes_oracle())
        _classes_lib.orc_last_error.restype = C.c_char_p
        _classes_lib.orc_last_error.argtypes = [C.c_void_p]
    return _classes_lib


class ClassesOracleProblem(OracleProblem):
    """an OracleProblem on the oracle with the size classes (and every explicit rule)"""

    def _open(self):
        self._lib = load_classes_oracle()
        self._h = C.c_void_p()
        rc = self._lib.orc_create(C.byref(self.spec.c), C.byref(self._h))
        if rc:
            msg = self._lib.orc_last_error(None).decode()
            raise {K.TO_EDIM: TO.DimensionMismatch, K.TO_EINVAL: TO.ArgumentError}.get(rc, TO.TrajOptError)(msg)


def on_class_oracle(build):
    """`build(cls)` with ClassesOracleProblem where the comparison helpers (parity_util.triple, test_gpu_solve.compare) ask for OracleProblem"""
    return lambda cls: build(ClassesOracleProblem if cls is OracleProblem else cls)


# ---- every op code in each class: the (4, 2) op programs on disjoint slices of x and u ------------------------------------------------
def ops_84(x, u):               # n = 8, m = 4: records op codes 0..19
    return transcendental(x[0:4], u[0:2]) + powers(x[4:7], [u[2] * u[3]]) + constant_rate([x[7], x[7]], [u[3]])[1:]


def ops_168(x, u):              # n = 15, m = 8: the largest state and control the class holds sit in the program's last slots
    return (transcendental(x[0:4], u[0:2]) + powers(x[4:7], [u[2]]) + constant_rate(x[7:9], u[3:4])
            + [x[9] * u[4] - x[10], TO.sin(x[11]) + u[5], x[12] * x[13] + u[6], TO.cos(x[14]) * u[7], x[10] + 0.1 * x[14], x[13] - u[7]])


CLASS_PROGRAMS = {"ops_84": (8, 4, ops_84), "ops_168": (15, 8, ops_168)}


def class_model(name, discrete=False):
    n, m, f = CLASS_PROGRAMS[name]
    return TO.AutodiffDynamics(n, m, f, discrete=discrete)


# ---- physical models --------------------------------------------------------------------------------------------------------------------
def quadrotor_function(mass=0.5, J=(0.0023, 0.0023, 0.004), gravity=(0.0, 0.0, -9.81), L=0.1750, kf=1.0, km=0.0245):
    """csrc/models.cuh dynamics<MODEL_QUADROTOR> without the relu on thrust (the recorder has none): equal to the built-in model for
    positive controls"""
    J1, J2, J3 = J
    gx, gy, gz = gravity
    inv_mass, iJ1, iJ2, iJ3 = 1.0 / mass, 1.0 / J1, 1.0 / J2, 1.0 / J3

    def f(x, u):
        qw, qx, qy, qz = x[3], x[4], x[5], x[6]
        wx, wy, wz = x[10], x[11], x[12]
        F1, F2, F3, F4 = kf * u[0], kf * u[1], kf * u[2], kf * u[3]
        Fz = F1 + F2 + F3 + F4
        vv = qx * qx + qy * qy + qz * qz
        ww = qw * qw - vv
        vr = qz * Fz
        Fwx = 2.0 * (qx * vr) + 2.0 * (qw * (qy * Fz))
        Fwy = 2.0 * (qy * vr) - 2.0 * (qw * (qx * Fz))
        Fwz = ww * Fz + 2.0 * (qz * vr)
        M1, M2, M3, M4 = km * u[0], km * u[1], km * u[2], km * u[3]
        t1, t2, t3 = L * (F2 - F4), L * (F3 - F1), (M1 - M2 + M3 - M4)
        Jw1, Jw2, Jw3 = J1 * wx, J2 * wy, J3 * wz
        return [x[7], x[8], x[9],
                -0.5 * (qx * wx + qy * wy + qz * wz),
                0.5 * (qw * wx + qy * wz - qz * wy),
                0.5 * (qw * wy + qz * wx - qx * wz),
                0.5 * (qw * wz + qx * wy - qy * wx),
                (mass * gx + Fwx) * inv_mass, (mass * gy + Fwy) * inv_mass, (mass * gz + Fwz) * inv_mass,
                (t1 - (wy * Jw3 - wz * Jw2)) * iJ1, (t2 - (wz * Jw1 - wx * Jw3)) * iJ2, (t3 - (wx * Jw2 - wy * Jw1)) * iJ3]
    return f


def planar_quadrotor_function(mass=1.0, J=0.01, arm=0.2, g=9.81):
    """x = [px, pz, theta, vx, vz, omega], u = [thrust 1, thrust 2]"""
    def f(x, u):
        s, c = TO.sin(x[2]), TO.cos(x[2])
        T = u[0] + u[1]
        return [x[3], x[4], x[5], -(T * s) * (1.0 / mass), (T * c) * (1.0 / mass) - g, (u[0] - u[1]) * (arm / J)]
    return f


def arm7_function(inertia=(1.0, 0.9, 0.8, 0.7, 0.6, 0.5, 0.4), damping=0.3, stiffness=0.5, coupling=0.2):
    """x = [q(7), qdot(7)], u = 7 joint torques: a damped chain with neighbour coupling through sin(q_i - q_{i+1})"""
    def f(x, u):
        q, qd = x[:7], x[7:]
        acc = []
        for i in range(7):
            a = u[i] - damping * qd[i] - stiffness * TO.sin(q[i])
            if i + 1 < 7:
                a = a - coupling * TO.sin(q[i] - q[i + 1])
            acc.append(a * (1.0 / inertia[i]))
        return list(qd) + acc
    return f


def quadrotor_model():
    return TO.AutodiffDynamics(13, 4, quadrotor_function())


def planar_quadrotor_model():
    return TO.AutodiffDynamics(6, 2, planar_quadrotor_function())


def arm7_model():
    return TO.AutodiffDynamics(14, 7, arm7_function())


def padded_closed_form(model, n, m):
    """the rows and columns of the padded (n x (n + m)) [A B] outside the model's own block: the unused state slots are carried as
    x+ = x + 0 by an explicit rule (identity) and set to zero by a jump map; no state depends on an unused control"""
    AB = np.eye(n, n + m) if not model.discrete else np.zeros((n, n + m))
    mask = np.ones((n, n + m), dtype=bool)
    mask[:model.n_out, :model.n] = False
    mask[:model.n_out, n:n + model.m] = False
    return AB, mask
