"""Dry run of the `-m gpu` tests with the CPU oracle standing in for the CUDA library on BOTH sides (so every comparison is trivially
equal): checks the Python-level flow of those tests (problem construction, argument validation, API calls) in a container without a GPU.
Not collected by pytest (no test_ prefix); the three tests that need the CUDA library itself are expected to fail, and
so are the to_create checks of test_gpu_dynamics_programs.py and its batches sized from the device's SM count.  Of
test_gpu_dispatch_boundaries.py, the landing tests (`to_kernel_choice`) are expected to fail; the library's row limits and the
per-instance tests (`to_set_model_params`, `to_set_goal_states`: no oracle counterpart) skip themselves, and the comparisons run at small
stand-in batch sizes.

    python tests/dryrun_gpu_tests_on_oracle.py
"""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
import trajopt_b200 as TO
import oracle_binding
import importlib
api = importlib.import_module(TO.Problem.__module__)
api.Problem = oracle_binding.OracleProblem
TO.Problem = oracle_binding.OracleProblem
import pytest
sys.exit(pytest.main(['--noconftest', '-W', 'ignore', os.path.join(ROOT, 'tests', 'test_gpu_parity.py'), os.path.join(ROOT, 'tests', 'test_gpu_fullsize.py'), os.path.join(ROOT, 'tests', 'test_golden.py'),
                  os.path.join(ROOT, 'tests', 'test_gpu_dynamics_programs.py'), os.path.join(ROOT, 'tests', 'test_gpu_dispatch_boundaries.py'), '-m', 'gpu', '-q', '-p', 'no:cacheprovider']))
