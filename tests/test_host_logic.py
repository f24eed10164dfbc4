"""CPU tests of the host side: the C-ABI library loads and exports every symbol include/*.h declares (no compute
calls without a GPU), the mirror API's host logic, and the multi-rank path (gloo, world_size 2)."""
import ctypes
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import trajopt_b200 as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(to_[a-z_0-9]+)\s*\(", hdr)))
    assert len(declared) >= 45
    lib = ctypes.CDLL(TO.capi.LIB_PATH)
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, f"libtrajopt_b200.so lacks {missing}"
    assert sorted(TO.capi.EXPORTED_SYMBOLS) == declared


def test_no_cpu_fallback_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    obj = TO.LQRObjective(np.eye(2), np.eye(1), np.eye(2), np.zeros(2), 5)
    with pytest.raises(TO.TrajOptError, match="no CPU fallback"):
        TO.Problem(TO.DoubleIntegrator(1), obj, np.zeros(2), 1.0)


def test_product_never_references_the_oracle():
    pkg = os.path.join(ROOT, "trajectoryoptimization.jl_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".jl")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "liboracle" not in text and "orc_" not in text and "oracle_binding" not in text, f


def test_constraint_list_and_objective_host_logic():
    n, m, N = 4, 1, 11
    cons = TO.ConstraintList(n, m, N)
    goal = TO.GoalConstraint(np.ones(n))
    bnd = TO.BoundConstraint(n, m, u_min=-1, u_max=1)
    TO.add_constraint(cons, bnd, (1, N - 1))
    TO.add_constraint(cons, goal, N)
    assert np.array_equal(TO.num_constraints(cons), [2] * (N - 1) + [n])      # src/constraint_list.jl:198-206
    assert [c for _, c in cons.zip()] == [bnd, goal] and list(cons.zip())[0][0] == (1, N - 1)
    with pytest.raises(TO.DimensionMismatch):                                   # src/constraint_list.jl:108-110
        TO.add_constraint(cons, TO.BoundConstraint(n + 1, m, u_min=-1, u_max=1), 1)
    c1 = TO.DiagonalCost(np.ones(n), np.ones(m))
    c2 = TO.QuadraticCost(np.eye(n), np.eye(m), H=np.ones((m, n)))
    s = c1 + c2                                                                 # +(c1, c2) src/cost_functions.jl:259-270
    assert isinstance(s, TO.QuadraticCost) and np.allclose(s.Q, 2 * np.eye(n)) and np.allclose(s.H, 1.0)
    obj = TO.Objective([c1] * (N - 1), c1)                                      # Objective(costs, cost_term) src/objective.jl:78-81
    assert len(obj) == N
    trk = TO.TrackingObjective(np.eye(n), np.eye(m), np.ones((N, n)), np.zeros((N - 1, m)))
    assert np.allclose(trk[3].q, -np.ones(n)) and trk[-1].terminal              # src/objective.jl:190-196
    assert TO.multi_gpu.shard_slice(10, 0, 4) == (0, 3) and TO.multi_gpu.shard_slice(10, 3, 4) == (8, 10)
    assert sum(b - a for a, b in (TO.multi_gpu.shard_slice(4096, r, 8) for r in range(8))) == 4096


def test_constraint_list_reference_test():
    """test/constraint_list.jl:33-78: add_constraint! order / insertion index, per-knot counts, copy, iteration, dimension check"""
    r = np.random.default_rng(2)
    n, m, N = 4, 1, 11
    cir = TO.CircleConstraint(n, [1.0, 1, 1], [1.0, 2, 3], [1.0, 1, 1])
    goal = TO.GoalConstraint(r.random(n))
    lin = TO.LinearConstraint(n, m, r.random((5, n)), r.random(5), TO.Inequality())
    bnd = TO.BoundConstraint(n, m, x_min=-r.random(n), x_max=r.random(n), u_min=-r.random(m), u_max=r.random(m))
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, cir, (1, N))
    assert cons.constraints[0] is cir and cons[0] is cir and cons.inds[0] == (1, N) and np.array_equal(cons.p, [cir.p] * N)     # :35-38
    TO.add_constraint(cons, goal, N)
    assert cons[1] is goal and cons.inds[1] == (N, N)                                                                            # :41-43
    assert np.array_equal(cons.p[:N - 1], [cir.p] * (N - 1)) and cons.p[-1] == cir.p + goal.p                                   # :44-45
    TO.add_constraint(cons, lin, (1, 4), 0)                                                                                      # add_constraint!(cons, lin, 1:4, 1)
    assert cons[0] is lin and cons[1] is cir and cons[-1] is goal and cons.inds[0] == (1, 4)                                    # :48-51
    assert np.array_equal(cons.p[:4], [cir.p + lin.p] * 4) and np.array_equal(cons.p[4:N - 1], [cir.p] * (N - 5)) and len(cons) == 3   # :52-54
    cons2 = cons.copy()
    TO.add_constraint(cons, bnd, (1, N - 1))
    assert len(cons) == 4 and len(cons2) == 3 and cons[-1] is bnd                                                               # :56-64
    assert TO.num_constraints(cons2) is not cons.p and not np.array_equal(TO.num_constraints(cons2), cons.p)
    with pytest.raises(TO.DimensionMismatch):                                                                                    # :67-68
        TO.add_constraint(cons, TO.LinearConstraint(2, 1, r.random((3, 2)), r.random(3), TO.Inequality()), (1, 4))
    assert [c for c in cons] == [lin, cir, goal, bnd] and [TO.output_dim(c) for c in cons] == [5, 3, n, 2 * (n + m)]             # :71-74


WORKER = textwrap.dedent("""
    import os, sys
    sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
    import numpy as np, torch, torch.distributed as dist
    import trajopt_b200 as TO
    from oracle_binding import OracleProblem
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:{port}", rank=int(sys.argv[1]), world_size=2)
    rank = dist.get_rank()
    B = 6
    lo, hi = TO.multi_gpu.shard_slice(B, rank, 2)
    full = TO.problems.cartpole(B=B, N=31, cls=OracleProblem, u_bound=3.0, goal=True)
    shard = TO.problems.cartpole(B=hi - lo, N=31, cls=OracleProblem, u_bound=3.0, goal=True)
    TO.set_initial_state(shard, full.x0[lo:hi]); TO.initial_controls(shard, TO.controls(full)[lo:hi])
    for p in (full, shard):
        TO.rollout(p); TO.ilqr_step(p, 2)
    g = TO.multi_gpu.global_merit(shard)            # SUM / MAX all-reduce over the two shards
    ref = np.array([TO.merit(full).sum(), TO.max_violation(full).max()])
    assert np.allclose(g.numpy(), ref, rtol=1e-12), (g, ref)
    assert np.allclose(TO.states(shard), TO.states(full)[lo:hi], rtol=0, atol=0)   # sharding does not change any instance
    dist.destroy_process_group()
    print("rank", rank, "ok")
""")


def test_two_rank_gloo_sharding_and_merit_allreduce(tmp_path):
    """the N>1 path on CPU: contiguous batch shards, no data-path collective, one SUM/MAX all-reduce of the merit."""
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, port=29000 + os.getpid() % 2000))
    procs = [subprocess.Popen([sys.executable, str(script), str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=240)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r} ok" in o, o


def test_live_problem_follows_mutations_of_objective_and_constraint_list():
    """the reference mutates a live problem in place -- set_LQR_goal!(prob.obj[k], xf), add_constraint!(get_constraints(prob), ...): the
    device-side tables are re-uploaded before the next call, and output buffers are sized from the current list (ADVICE r01)."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from oracle_binding import OracleProblem
    import trajopt_b200 as TO
    n, m, N = 4, 2, 11
    xf = np.array([0, 2.0, 0, 0])
    obj = TO.LQRObjective(np.eye(n), np.eye(m), np.eye(n) * 10, xf, N)
    cons = TO.ConstraintList(n, m, N)
    TO.add_constraint(cons, TO.GoalConstraint(xf), N)
    prob = OracleProblem(TO.DoubleIntegrator(2), obj, np.zeros(n), 1.0, xf=xf, constraints=cons)
    TO.initial_controls(prob, np.ones((1, N - 1, m))); TO.rollout(prob)
    J0 = TO.cost(prob)[0]
    xg = np.array([1.0, -1.0, 0, 0])
    for k in range(N):
        TO.set_LQR_goal(prob.obj[k], xg)
    J1 = TO.cost(prob)[0]
    ref = OracleProblem(TO.DoubleIntegrator(2), prob.obj.copy(), np.zeros(n), 1.0, xf=xf, constraints=cons.copy())
    TO.initial_controls(ref, np.ones((1, N - 1, m))); TO.rollout(ref)
    assert J1 != J0 and np.isclose(J1, TO.cost(ref)[0], rtol=1e-14)
    np.testing.assert_array_equal(TO.states(prob), TO.states(ref))          # the trajectory survived the re-upload
    bnd = TO.BoundConstraint(n, m, u_min=-0.5, u_max=0.5)
    TO.add_constraint(TO.get_constraints(prob), bnd, (1, N - 1), idx=0)
    vals = TO.evaluate_constraints(prob, 0)
    assert vals.shape == (1, N - 1, 4) and np.allclose(vals[0, :, :2], 0.5) and np.allclose(vals[0, :, 2:], -1.5)
    assert TO.evaluate_constraints(prob, 1).shape == (1, 1, n)
    TO.set_options(prob, penalty_scaling=3.0); TO.set_options(prob, iterations_linesearch=7)
    assert prob._options.penalty_scaling == 3.0 and prob._options.iterations_linesearch == 7      # earlier settings are kept
    prob.close(); ref.close()


def test_abi_struct_layout_matches_the_binding_tables():
    """INTEGRATION.md's offset table (what a Julia / ctypes binding has to reproduce field for field) against offsetof / sizeof printed by a C
    program compiled from include/trajopt_b200.h, and against the ctypes structures of the Python binding."""
    import re
    import subprocess
    import tempfile
    import ctypes
    import trajopt_b200 as TO
    hdr = open(os.path.join(ROOT, "include", "trajopt_b200.h")).read()
    structs = {}
    for body, name in re.findall(r"typedef struct \{(.*?)\}\s*(to_cost_spec|to_dynamics_spec|to_constraint_spec|to_spec|to_options);", hdr, flags=re.S):
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            names = decl.split(",")
            first = names[0].split()[-1]
            fields.append(first.lstrip("*"))
            fields += [n.strip().lstrip("*") for n in names[1:]]
        structs[name] = fields
    src = "#include <stdio.h>\n#include <stddef.h>\n#include \"trajopt_b200.h\"\nint main() {\n"
    for name, fields in structs.items():
        for f in fields:
            src += f'  printf("{name} {f} %zu\\n", offsetof({name}, {f}));\n'
        src += f'  printf("{name} sizeof %zu\\n", sizeof({name}));\n'
    src += "  return 0;\n}\n"
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "l.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "l.c"), "-o", os.path.join(d, "l")])
        out = subprocess.check_output([os.path.join(d, "l")], text=True)
    c_layout = {tuple(l.split()[:2]): int(l.split()[2]) for l in out.splitlines()}
    # the table in INTEGRATION.md: rows `| to_spec | field | offset | ...`
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    table = {(m.group(1), m.group(2)): int(m.group(3)) for m in re.finditer(r"^\| `(to_\w+)` \| `(\w+)` \| (\d+) \|", doc, flags=re.M)}
    assert table, "INTEGRATION.md has no struct layout table"
    assert table == c_layout, {k: (table.get(k), c_layout.get(k)) for k in set(table) | set(c_layout) if table.get(k) != c_layout.get(k)}
    # the ctypes mirror
    for name in structs:
        cls = getattr(TO.capi, name)
        assert ctypes.sizeof(cls) == c_layout[(name, "sizeof")], name
        for f in structs[name]:
            assert getattr(cls, f).offset == c_layout[(name, f)], (name, f)


def test_environment_switches_read_are_exactly_the_documented_ones():
    """The TO_* variables the CUDA sources read with getenv are exactly the TO_* rows of INTEGRATION.md's switch table (a switch a
    maintainer cannot find is a trap, a documented one the library ignores misleads), and exactly the three kept for profiling and A/B."""
    import glob
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = set()
    for f in glob.glob(os.path.join(root, "trajectoryoptimization.jl_b200", "csrc", "*.cu*")):
        names |= set(re.findall(r'getenv\("(TO_[A-Z0-9_]+)"\)', open(f).read()))
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    section = doc[doc.index("## Environment switches of the library"):]
    section = section[:section.index("\n## ")] if "\n## " in section else section
    rows = set()
    for line in section.splitlines():
        if line.startswith("| `"):
            rows |= set(re.findall(r"`(TO_[A-Z0-9_]+)", line.split("|")[1]))
    assert names == rows, f"read but not documented: {sorted(names - rows)}; documented but not read: {sorted(rows - names)}"
    assert names == {"TO_NO_OVERLAP", "TO_NO_FRAG", "TO_EXPAND_SEEDS"}, sorted(names)
