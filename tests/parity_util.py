"""Conditioning-aware GPU-vs-oracle comparison (test infrastructure).

Why: the closed loop of the BASELINE Quadrotor problem amplifies rounding differences by orders of magnitude per stage (cheap controls
R = 0.01 against Qf = 100, a 5 s horizon whose open-loop initial guess tumbles): a relative difference of 1e-11 in the gains of one
backward pass is 1e-7 in the trajectory after the forward pass and O(1e-2) three iterations later, for ANY two fp64 implementations
(Cartpole / Acrobot agree to 1e-11 after six iterations).  So:

  * ONE kernel application on identical inputs is compared with the oracle at kernel tolerance, the oracle running the arithmetic
    form of the backward pass that the CUDA kernel uses (oracle_binding.match_algebra; the two forms themselves agree to 1e-11);
  * everything DOWNSTREAM of a backward pass is compared against a yardstick: the TWIN, the same oracle whose backward passes return
    gains perturbed by the relative amount GAIN_TOL (= the kernel tolerance of the gains; oracle.hpp Options::gain_noise).  The
    divergence D_b of twin and oracle on instance b is what a backward pass that is accurate to GAIN_TOL may do to that instance; the CUDA
    result has to stay within FACTOR x D_b (or the tight tolerance, whichever is larger).  Discrete decisions (step sizes, restarts)
    are compared on the instances where the perturbation does not flip them in the twin."""
import numpy as np

import trajopt_b200 as TO
from oracle_binding import OracleProblem, match_algebra

GAIN_TOL = 2e-9     # kernel tolerance of K, d (measured: 4e-11 full-state kernel, 1.4e-9 register-resident kernel on random attitudes)
FACTOR = 5.0


def inst_err(a, b):
    """per-instance max |a - b| / max(1, max |b|)   (arrays with the batch on axis 0)"""
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    B = b.shape[0]
    d = np.abs(a - b).reshape(B, -1).max(axis=1) if b.size else np.zeros(B)
    s = np.maximum(1.0, np.abs(b).reshape(B, -1).max(axis=1)) if b.size else np.ones(B)
    d = np.where(np.isfinite(d), d, np.inf)
    return d / s


def triple(build, opts=None):
    """(cuda problem, oracle in the same arithmetic form, twin = that oracle with GAIN_TOL noise on the gains of every backward pass)"""
    g = build(TO.Problem)
    if opts:
        TO.set_options(g, **opts)
    o = match_algebra(g, build(OracleProblem))
    t = match_algebra(g, build(OracleProblem)).set_gain_noise(GAIN_TOL)
    return g, o, t


def triple_with_options(build, opts=None):
    """`triple` with SOLVER options (regularisation, line search, AL schedule) applied to all three problems; `backward_kernel` is a kernel
    choice of the CUDA problem and goes to it alone (the oracle has one backward pass, in the arithmetic form match_algebra picks)"""
    opts = dict(opts or {})
    kernel = opts.pop("backward_kernel", None)
    g = build(TO.Problem)
    TO.set_options(g, **opts, **({} if kernel is None else {"backward_kernel": kernel}))
    o = match_algebra(g, build(OracleProblem))
    t = match_algebra(g, build(OracleProblem)).set_gain_noise(GAIN_TOL)
    for p in (o, t):
        TO.set_options(p, **opts)
    return g, o, t


def check(what, a_gpu, a_orc, a_twin, tight, sel=None, outliers=0.0):
    """every instance (but a fraction `outliers` of them -- after several closed-loop iterations of a chaotic instance one noise draw of the
    twin is a coarse yardstick): err(gpu, oracle) <= max(tight, FACTOR * err(twin, oracle)); returns (worst gpu error, worst twin error)"""
    e, d = inst_err(a_gpu, a_orc), inst_err(a_twin, a_orc)
    if sel is not None:
        e, d = e[sel], d[sel]
    tol = np.maximum(tight, FACTOR * d)
    bad = np.nonzero(~(e <= tol))[0]
    assert bad.size <= outliers * e.size, (f"{what}: {bad.size} of {e.size} instances outside the budget; worst gpu-vs-oracle {e[bad].max():.3e} "
                           f"with twin divergence {d[bad][np.argmax(e[bad])]:.3e} (tight tolerance {tight:.0e})")
    return float(e.max()) if e.size else 0.0, float(d.max()) if d.size else 0.0


def decisions_agree(what, v_gpu, v_orc, v_twin, sel=None, allow=0.0):
    """discrete per-instance results are compared where the perturbed twin takes the oracle's decision; `allow`: tolerated fraction of
    mismatches among those (a decision that sits within the GAIN_TOL band of its threshold for the cuda run but not for the twin's noise draw)"""
    v_gpu, v_orc, v_twin = np.asarray(v_gpu), np.asarray(v_orc), np.asarray(v_twin)
    m = (v_orc == v_twin)
    if sel is not None:
        m &= sel
    bad = int(np.sum(v_gpu[m] != v_orc[m]))
    assert bad <= allow * max(1, int(m.sum())), f"{what}: {bad} mismatches among {int(m.sum())} decidable instances"
    return m & (v_gpu == v_orc)
