"""CPU checks of the register-resident Riccati formulation (csrc/riccati_frag.cu, csrc/frag_layout.cuh):
the lane-level NumPy emulation of the kernel's MMA-fragment algebra (frag_emulator.py) reproduces the dense recursion,
and the index tables compiled into the CUDA sources are the ones the emulation uses."""
import os
import subprocess
import tempfile

import numpy as np

import frag_emulator as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fragment_recursion_matches_dense_recursion():
    rng = np.random.default_rng(0)
    HN = rng.standard_normal((12, 12)); HN = HN @ HN.T + np.eye(12)
    gN = rng.standard_normal(12)
    Sacc = FE.terminal_state(HN, gN)
    S, s = HN.copy(), gN.copy()
    for k in range(8):
        rho = [0.0, 0.3, 2.0][k % 3]
        AB = 0.4 * rng.standard_normal((12, 16))
        H = np.diag(rng.uniform(0.1, 1, 16)); blk = rng.standard_normal((3, 3)); H[3:6, 3:6] += blk @ blk.T
        g = rng.standard_normal(16)
        Sacc, K, d, t1, t2, ok = FE.knot(Sacc, AB, H, g, rho, symmetrise_diag=(k % 4 == 0))
        Ssym = FE.matrix_from_frag(Sacc)
        assert np.array_equal(Ssym[:8, 8:], Ssym[8:, :8].T)                # the off-diagonal tiles are exact mirrors
        S, s, Kr, dr, r1, r2 = FE.dense_reference(S, s, AB, H, g, rho)
        Sh = FE.matrix_from_frag(Sacc)
        Sf = np.array([[Sh[FE.PHYS_X[e], FE.PHYS_X[f]] for f in range(12)] for e in range(12)])
        sf = np.array([Sh[0, FE.PHYS_X[e]] for e in range(12)])
        scale = np.abs(S).max()
        assert ok
        assert np.abs(Sf - S).max() < 1e-12 * scale and np.abs(sf - s).max() < 1e-12 * scale
        sc = np.array([Sh[FE.PHYS_X[e], 0] for e in range(12)])            # column 0 carries s as well (s = Qx + W'd)
        assert np.abs(sc - s).max() < 1e-12 * scale
        assert np.abs(K - Kr).max() < 1e-12 * max(1, np.abs(Kr).max()) and np.abs(d - dr).max() < 1e-12 * max(1, np.abs(dr).max())
        assert abs(t1 - r1) < 1e-12 * max(1, abs(r1)) and abs(-0.5 * (t1 + rho * t2) - r2) < 1e-12 * max(1, abs(r2))


def test_block_inverse_of_the_kernel():
    """(Quu + rho I)^-1 by 2 x 2 block elimination, the formulas of k_riccati_frag, against numpy.linalg.inv"""
    rng = np.random.default_rng(3)
    for _ in range(50):
        A = rng.standard_normal((4, 4)); M = A @ A.T + 0.05 * np.eye(4)
        a, bq, c = M[0, 0], M[0, 1], M[1, 1]
        M20, M30, M21, M31 = M[0, 2], M[0, 3], M[1, 2], M[1, 3]
        R00, R01, R11 = M[2, 2], M[2, 3], M[3, 3]
        detP = a * c - bq * bq; iP = 1 / detP
        yt00, yt01 = M20 * c - M21 * bq, M21 * a - M20 * bq
        yt10, yt11 = M30 * c - M31 * bq, M31 * a - M30 * bq
        z00, z01, z11 = yt00 * M20 + yt01 * M21, yt00 * M30 + yt01 * M31, yt10 * M30 + yt11 * M31
        s00, s01, s11 = R00 - iP * z00, R01 - iP * z01, R11 - iP * z11
        detS = s00 * s11 - s01 * s01; iS = 1 / detS
        v00, v01, v11 = s11 * iS, -s01 * iS, s00 * iS
        y00, y01, y10, y11 = yt00 * iP, yt01 * iP, yt10 * iP, yt11 * iP
        n00, n01 = -(v00 * y00 + v01 * y10), -(v00 * y01 + v01 * y11)
        n10, n11 = -(v01 * y00 + v11 * y10), -(v01 * y01 + v11 * y11)
        p00 = c * iP - (y00 * n00 + y10 * n10); p01 = -bq * iP - (y00 * n01 + y10 * n11); p11 = a * iP - (y01 * n01 + y11 * n11)
        Minv = np.array([[p00, p01, n00, n10], [p01, p11, n01, n11], [n00, n01, v00, v01], [n10, n11, v01, v11]])
        ref = np.linalg.inv(M)
        assert np.abs(Minv - ref).max() < 1e-10 * np.abs(ref).max()
        assert a > 0 and detP > 0 and s00 > 0 and detS > 0          # the kernel's positive-definiteness test on an SPD matrix
    Mi = np.diag([1.0, 1.0, -0.5, 1.0])                            # indefinite: a leading minor of the Schur complement is negative
    assert not (Mi[2, 2] > 0)


def test_cuda_index_tables_match_the_emulation():
    src = r'''
#include <cstdio>
#define __host__
#define __device__
#include "frag_layout.cuh"
int main() {
    for (int j = 0; j < 16; j++) printf("%d ", fraglayout::phys_z(j));
    printf("\n");
    for (int p = 0; p < 16; p++) printf("%d ", fraglayout::e_of_p(p));
    printf("\n");
    for (int e = 0; e < 12; e++) for (int j = 0; j < 16; j++) printf("%d ", fraglayout::ab_index(e, j));
    printf("\n%d %d %d %d\n", TO_REC_LEN, TO_REC_G, TO_REC_HD, TO_REC_HB);
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.cpp"), "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", "-x", "c++", "-I", os.path.join(ROOT, "trajectoryoptimization.jl_b200", "csrc"), os.path.join(d, "t.cpp"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True).splitlines()
    phys = [int(v) for v in out[0].split()]
    assert phys == FE.PHYS
    e_of_p = [int(v) for v in out[1].split()]
    assert e_of_p == [FE.PHYS_X.index(p) if p in FE.PHYS_X else -1 for p in range(16)]
    idx = np.array([int(v) for v in out[2].split()]).reshape(12, 16)
    assert sorted(idx.ravel()) == list(range(192))                       # a permutation of the fragment block
    AB = np.arange(192, dtype=float).reshape(12, 16)
    abf = FE.ab_fragments(AB)                                            # abf[ks][mi][lane]
    rec = np.zeros(192)
    for e in range(12):
        for j in range(16):
            rec[idx[e, j]] = AB[e, j]
    for ks in range(3):
        for lane in range(32):
            for mi in range(2):
                assert rec[(ks * 32 + lane) * 2 + mi] == abf[ks, mi, lane]
    assert [int(v) for v in out[3].split()] == [240, 192, 208, 224]
    # the nibble table of k_expand_lie_rec
    tab = 0x6420FDB9E7CA8531
    assert [(tab >> (4 * j)) & 15 for j in range(16)] == FE.PHYS
