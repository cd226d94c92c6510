"""Cases of the many_vs_many tests shared by the emulated checks (tests/host_emul/many_vs_many_checks.py) and the GPU
tests (tests/test_gpu_many_vs_many.py): a brute force of the counts with np.intersect1d, and a database with empty rows
and the keys 0 and 2^64 - 1 against identical, nested, empty and non-matching queries."""
import numpy as np

from tests.multigather_cases import workload

BIG = np.uint64(2**64 - 1)


def brute(queries, rows):
    "|query ∩ row| for every (query, row): a (len(queries), len(rows)) uint32 array"
    return np.array([[len(np.intersect1d(q, r)) for r in rows] for q in queries], dtype=np.uint32).reshape(
        len(queries), len(rows))


def cases():
    "database rows and queries: shared, identical and nested queries, an empty one between them, keys 0 and 2^64 - 1"
    rows, queries = workload()
    rows = rows[:120] + [np.zeros(0, np.uint64), np.array([0, 5, BIG], np.uint64), np.zeros(0, np.uint64)]
    qs = [queries[0], queries[0].copy(), queries[0][::2].copy(), np.zeros(0, np.uint64), queries[3],
          np.array([0, BIG], np.uint64), queries[1], queries[5], queries[4]]
    return rows, qs
