#!/usr/bin/env python
"""Moderate ExecuteScalarExpression calls that reach every op of expr_eval_kernel (every function of the random trees of
tests/test_gpu_expression.py, BOOL outputs, null literals, failing programs, a tree split into several programs,
sliced columns and tables of many chunks), for compute-sanitizer memcheck and racecheck:

    compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/lab/san_expr.py
    compute-sanitizer --tool racecheck --error-exitcode 9 python scripts/lab/san_expr.py

Every result is compared with both oracles of the test file (node by node through CallFunction, and the
exec_model fold), so a sanitizer-clean run is also a correct one."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import exec_model as M  # noqa: E402
import test_gpu_expression as T  # noqa: E402
from arrow_go_b200 import compute as pc  # noqa: E402


def main():
    trees = 0
    for n, table in ((1, False), (1500, False), (2500, True)):
        rng = T._rng("san", n, table)
        types = [pc.INT32, pc.FLOAT64, pc.INT8, pc.UINT64]
        cols = [T.column(rng, t, n, table) for t in types]
        for vals in (T.values, T.small_values):
            for _ in range(12):
                T.check(T.random_tree(rng, types, int(rng.integers(1, 5)), vals), cols, table)
                trees += 1
    rng = T._rng("san-wide")
    cols = [T.column(rng, pc.FLOAT64 if j % 2 else pc.INT32, 2000, True) for j in range(20)]

    def full(d, k):
        if d == 0:
            return ("field", k % 20)
        return ("call", "add_unchecked" if d % 2 else "multiply_unchecked", [full(d - 1, 2 * k), full(d - 1, 2 * k + 1)], None)

    T.check(full(9, 0), cols, True)   # more registers and columns than one program holds
    trees += 1
    print(f"san_expr ok: {trees} trees, every result matched both oracles ({len(M.NUMERIC)} numeric types)")


if __name__ == "__main__":
    main()
