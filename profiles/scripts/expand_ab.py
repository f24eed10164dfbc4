"""A/B of the record-path dynamics-expansion kernels: dump the [A_e B_e] blocks after to_expand, and the gains, trajectory and merit after
iLQR iterations whose expansions run as the overlapped mode 1 / mode 2 launches (the late instances through the compact late list).
usage: expand_ab.py out.npz   (TO_EXPAND_V1=1 selects k_expand_lie, default k_expand_lie_rec); compare two dumps with --cmp a.npz b.npz
Arrays above 64 MB are stored as their SHA-256 digest plus a strided sample."""
import hashlib
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if sys.argv[1] == "--cmp":
    a, b = np.load(sys.argv[2]), np.load(sys.argv[3])
    worst = 0.0
    for k in a.files:
        d = float(np.max(np.abs(a[k].astype(float) - b[k].astype(float)))) if a[k].size else 0.0
        worst = max(worst, d)
        print(f"{k:16s} max|a-b| = {d:.3e}  identical={np.array_equal(a[k], b[k])}")
    print("A/B", "IDENTICAL" if worst == 0.0 else f"DIFFER (max {worst:.3e})")
    sys.exit(0)
import trajopt_b200 as TO

out = {}


def put(key, arr):
    arr = np.ascontiguousarray(arr)
    if arr.nbytes > 64 << 20:
        out[key + "_sha256"] = np.frombuffer(hashlib.sha256(arr.tobytes()).digest(), dtype=np.uint8)
        out[key + "_sample"] = arr.reshape(-1)[::97].copy()
    else:
        out[key] = arr


# to_expand (mode 0) at the benchmark size and at sizes that leave partial knot blocks
for (B, N) in ((4096, 101), (1, 2), (3, 5), (33, 2), (2, 64), (5, 23)):
    p = TO.problems.quadrotor(B=B, N=N, error_state=True)
    TO.rollout(p)
    TO.expand(p)
    put(f"ABe_{B}_{N}", TO.error_dynamics(p))
    p.close()

# iLQR iterations: iteration 1 expands every instance, the later ones run the overlapped launches (mode 1 on the main stream, mode 2 for the
# instances the first line-search pass did not accept).  The gains are the Riccati pass's function of the records those launches wrote.
for (B, N) in ((4096, 101), (37, 101), (5, 23)):
    p = TO.problems.quadrotor(B=B, N=N, error_state=True)
    TO.rollout(p)
    for it in range(3):
        TO.ilqr_step(p, 2 if it == 0 else 1)
        K, d = TO.gains(p)
        put(f"K{it}_{B}_{N}", K); put(f"d{it}_{B}_{N}", d)
        put(f"X{it}_{B}_{N}", TO.states(p)); put(f"J{it}_{B}_{N}", TO.merit(p))
    TO.expand(p)
    put(f"ABe_it_{B}_{N}", TO.error_dynamics(p))
    p.close()
np.savez(sys.argv[1], **out)
print("wrote", sys.argv[1])
