"""Covering-array properties of the suite's flag matrices (test_flag_matrix.py, test_vanilla_flags.py)."""
from itertools import combinations


def assert_covers_every_pair(matrix, dims):
    """every value of every row lies in its dimension, and every pair of values of any two dimensions appears in
    some row"""
    for row in matrix:
        assert len(row) == len(dims), row
        for v, dim in zip(row, dims):
            assert v in dim, (row, v)
    missing = []
    for i, j in combinations(range(len(dims)), 2):
        seen = {(r[i], r[j]) for r in matrix}
        missing += [(i, a, j, b) for a in dims[i] for b in dims[j] if (a, b) not in seen]
    assert not missing, missing
