"""NumPy restatement of the lane / block algebra of the record cost-expansion kernel k_expansion_rec16b (csrc/rollout.cu) -- test infrastructure,
like frag_emulator.py.  It runs the kernel's ALGORITHM on the CPU: the host-built term table (capi.cu upload_exptab: packed knot range, rows per
knot, multiplier index of the row at knot 0), blocks of 16 knots per 16-lane group, the 16-bit activity mask of a term inside a block, the
multiplier pointer of the block's first knot, phase A (state entries), phase B (attitude projection by lane j for knot j), phase C (control
entries), and the 48-double image [g~ | hd | Hb] of the record in the physical order of frag_layout.cuh.  tests/test_costexp_emulator.py
compares the images with the oracle's dense error-state expansion (Altro error_expansion!, oracle/oracle.hpp)."""
import numpy as np

QS, N_X, N_U = 3, 13, 4
MAXT = 3


def phys_x(e):                                   # frag_layout.cuh
    return [1, 3, 5, 8, 10, 12, 7, 14, 9, 11, 13, 15][e]


def phys_z(j):
    return phys_x(j) if j < 12 else 2 * (j - 12)


def build_term_table(cons, mus, n=N_X, m=N_U):
    """capi.cu upload_exptab.  cons: list of (constraint, first, last) with 1-based knot ranges, in ConstraintList order; mus: penalties.
    -> per z entry a list of <= MAXT terms (pkx, pky, nms, bound) with the kernel's packing, and the multiplier offsets of the constraints."""
    nm = n + m
    offsets, off = [], 0
    for (c, first, last) in cons:
        offsets.append(off); off += (last - first + 1) * c.p
    table = [[] for _ in range(nm)]
    for i in range(nm):
        for ci, (c, first, last) in enumerate(cons):
            kind = "BoundConstraint" if hasattr(c, "z_max") else type(c).__name__      # (StateBound / ControlBound included)
            mu = mus[ci]
            for side in range(2):
                row, sign, bound, eq = -1, 1.0, 0.0, False
                if kind == "GoalConstraint":
                    if side == 0 and i < n and (i + 1) in list(c.inds):
                        row = list(c.inds).index(i + 1); bound = c.xf[row]; eq = True
                elif kind == "BoundConstraint":
                    fin_max, fin_min = np.isfinite(c.z_max), np.isfinite(c.z_min)
                    if side == 0 and fin_max[i]:
                        row = int(fin_max[:i].sum()); bound = c.z_max[i]
                    if side == 1 and fin_min[i]:
                        row = int(fin_max.sum() + fin_min[:i].sum()); bound = c.z_min[i]; sign = -1.0
                else:
                    raise ValueError("the record path takes Goal / Bound constraints only")
                if row < 0:
                    continue
                assert len(table[i]) < MAXT and first < 4095 and c.p < 128
                pkx = first | ((last - first) << 12) | (c.p << 24) | ((1 << 31) if eq else 0)
                pky = (offsets[ci] + row - first * c.p) & 0xFFFFFFFF          # unsigned wrap-around, as in the kernel
                table[i].append((pkx, pky, -mu * sign, bound))
    return table, offsets, off


def block_images(X, U, lam_flat, table, cost_of_knot, costs, N):
    """one instance: X [N, 13], U [N-1, 4], lam_flat [lambda_len]; costs[c] = (Qd[13], q[13], Rd[4], r[4]); -> image [N, 48]."""
    n, m = N_X, N_U
    out = np.zeros((N, 48))
    for kb in range(0, N, 16):
        nk = min(16, N - kb)
        att = np.zeros((16, 12))
        # ---- phase A: lane i = state entry x_i, 16 steps -----------------------------------------------------------------------
        for i in range(n):
            terms = table[i]
            act, lp, ls = [], [], []
            for (pkx, pky, nms, bnd) in terms:
                first, span = pkx & 0xFFF, (pkx >> 12) & 0xFFF
                lo, hi = max(first - 1 - kb, 0), min(first + span - kb, nk)
                act.append(((0xFFFF >> (16 - (hi - lo))) << lo) if hi > lo else 0)
                ls.append((pkx >> 24) & 0x7F)
                v = (pky + (kb + 1) * ls[-1]) & 0xFFFFFFFF
                lp.append(v - (1 << 32) if v >= (1 << 31) else v)           # (int) of the unsigned sum: may point before the block's first row
            e = i if i < QS else i - 1
            for kk in range(nk):
                k = kb + kk
                Qd, q, _, _ = costs[cost_of_knot[k]]
                zi = X[k, i]
                g, h = Qd[i] * zi + q[i], Qd[i]
                for t, (pkx, pky, nms, bnd) in enumerate(terms):
                    if (act[t] >> kk) & 1:
                        lb = nms * (zi - bnd) + lam_flat[lp[t] + kk * ls[t]]
                        if (pkx >> 31) or lb <= 0.0:
                            g += -lb if nms < 0.0 else lb
                            h += abs(nms)
                if QS <= i <= QS + 3:
                    att[kk, 3 * (i - QS):3 * (i - QS) + 3] = (g, h, zi)
                else:
                    p = phys_x(e)
                    out[k, p] = g; out[k, 16 + p] = h
                    if e == 7:
                        out[k, 32 + 12:32 + 16] = (0.0, 0.0, 0.0, h)
        # ---- phases B and C: lane j = knot kb + j -------------------------------------------------------------------------------------
        for j in range(nk):
            k = kb + j
            gq, hq, q = att[j, 0::3], att[j, 1::3], att[j, 2::3]
            G = np.array([[-q[1], q[0], q[3], -q[2]], [-q[2], -q[3], q[0], q[1]], [-q[3], q[2], -q[1], q[0]]])     # rows of (L(q) H)'
            qb = float(q @ gq)
            for cc in range(3):
                ge = float(G[cc] @ gq)
                hb = [float((G[cc] * hq) @ G[c2]) for c2 in range(3)]
                hd = hb[cc] - qb
                p = 8 + 2 * cc
                out[k, p] = ge; out[k, 16 + p] = hd
                row = [hd if c2 == cc else hb[c2] for c2 in range(3)] + [0.0]
                out[k, 32 + 4 * cc:32 + 4 * cc + 4] = row
            _, _, Rd, r = costs[cost_of_knot[k]]
            for a in range(m):
                g = h = 0.0
                if k != N - 1:
                    z = U[k, a]
                    g, h = Rd[a] * z + r[a], Rd[a]
                    for (pkx, pky, nms, bnd) in table[n + a]:
                        if 0 <= (k + 1) - (pkx & 0xFFF) <= ((pkx >> 12) & 0xFFF):
                            idx = (pky + (k + 1) * ((pkx >> 24) & 0x7F)) & 0xFFFFFFFF
                            lb = nms * (z - bnd) + lam_flat[idx]
                            if (pkx >> 31) or lb <= 0.0:
                                g += -lb if nms < 0.0 else lb
                                h += abs(nms)
                out[k, 2 * a] = g; out[k, 16 + 2 * a] = h
    return out


def image_from_dense(g, H):
    """the 48-double image of a dense error-state expansion (g [16], H [16, 16], logical order x_e then u) + the entries it cannot hold"""
    img = np.zeros(48)
    P = [phys_z(j) for j in range(16)]
    for j in range(16):
        img[P[j]] = g[j]; img[16 + P[j]] = H[j, j]
    J = [3, 4, 5, 7]                                   # logical coordinates on the physical slots 8, 10, 12, 14
    for a in range(4):
        for b in range(4):
            img[32 + 4 * a + b] = H[J[a], J[b]]
    rest = H.copy()
    rest[np.diag_indices(16)] = 0.0
    for a in J:
        for b in J:
            rest[a, b] = 0.0
    return img, float(np.max(np.abs(rest)))
