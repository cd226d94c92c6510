#!/usr/bin/env python
"""Golden vectors for the ANI / distance estimators (SURVEY §8 f4).

distance_utils.py of the reference is plain Python (scipy + numpy), so unlike the Rust core it CAN
be executed without a Rust toolchain: this script imports <checkout>/src/sourmash/
distance_utils.py by path (with a stub for its `.logging` import; nothing else of the package is
needed) and records its outputs on a grid of inputs.  The result is committed as
golden_ani.json; tests/test_distance_utils.py compares sourmash_b200.distance_utils with it
bit-for-bit.  Run once:  SMB_REFERENCE=<sourmash checkout> python tests/golden/make_golden_ani.py
"""
import importlib.util
import itertools
import json
import os
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle.reference import checkout  # noqa: E402

REF = os.path.join(checkout(), "src", "sourmash")
HERE = os.path.dirname(os.path.abspath(__file__))

pkg = types.ModuleType("refsourmash")
pkg.__path__ = [REF]
sys.modules["refsourmash"] = pkg
log = types.ModuleType("refsourmash.logging")
log.notify = lambda *a, **k: None
sys.modules["refsourmash.logging"] = log
spec = importlib.util.spec_from_file_location("refsourmash.distance_utils", os.path.join(REF, "distance_utils.py"))
du = importlib.util.module_from_spec(spec)
sys.modules["refsourmash.distance_utils"] = du
spec.loader.exec_module(du)

out = {"source": "sourmash distance_utils.py (reference commit 6ae9cd32), scipy %s" % __import__("scipy").__version__}

rows = []
for j, k, scaled, n in itertools.product([0.0, 1.0, 1e-4, 0.0123, 0.3206949023586102, 0.5, 0.97, 0.999999],
                                          [7, 21, 31, 51], [1, 100, 1000], [50, 5000, 5_000_000]):
    try:
        r = du.jaccard_to_distance(j, k, scaled, n_unique_kmers=n)
        rows.append({"in": [j, k, scaled, n], "dist": r.dist, "p": r.p_nothing_in_common, "err": r.jaccard_error,
                     "p_exc": r.p_exceeds_threshold, "je_exc": r.je_exceeds_threshold, "ani": r.ani})
    except ValueError as e:
        rows.append({"in": [j, k, scaled, n], "error": str(e)})
out["jaccard_to_distance"] = rows

rows = []
for c, k, scaled, n, ci in itertools.product([0.0, 1.0, 1e-3, 0.1, 0.4828, 0.9, 0.9999], [7, 21, 31, 51],
                                             [1, 100, 1000], [1000, 5_177_000], [False, True]):
    try:
        r = du.containment_to_distance(c, k, scaled, n_unique_kmers=n, estimate_ci=ci)
        rows.append({"in": [c, k, scaled, n, ci], "dist": r.dist, "p": r.p_nothing_in_common, "lo": r.dist_low,
                     "hi": r.dist_high, "p_exc": r.p_exceeds_threshold, "ani": r.ani, "ani_low": r.ani_low,
                     "ani_high": r.ani_high})
    except ValueError as e:
        rows.append({"in": [c, k, scaled, n, ci], "error": str(e)})
out["containment_to_distance"] = rows

out["set_size_exact_prob"] = [{"in": [s, sc, re], "p": float(du.set_size_exact_prob(s, sc, relative_error=re))}
                              for s, sc, re in itertools.product([10, 1000, 20000, 5_177_000, 10**8], [1, 10, 1000],
                                                                 [0.05, 0.2])]
out["set_size_chernoff"] = [{"in": [s, sc, re], "p": float(du.set_size_chernoff(s, sc, relative_error=re))}
                            for s, sc, re in itertools.product([1000, 5_177_000], [10, 1000], [0.05, 0.2])]
rows = []
for L, k, r1 in itertools.product([10, 5000, 10**7], [2, 21, 51], [0.0, 1e-6, 0.01, 0.2, 0.9]):
    try:
        rows.append({"in": [L, k, r1], "v": du.var_n_mutated(L, k, r1)})
    except ValueError as e:                                # tiny inputs: the formula goes negative
        rows.append({"in": [L, k, r1], "error": str(e)})
out["var_n_mutated"] = rows
out["p_nothing_common"] = [{"in": [m, k, sc, n], "p": du.get_exp_probability_nothing_common(m, k, sc, n_unique_kmers=n)}
                           for m, k, sc, n in itertools.product([0.0, 1.0, 0.001, 0.05, 0.3], [21, 31], [1, 1000],
                                                                [100, 10**6])]
with open(os.path.join(HERE, "golden_ani.json"), "w") as fh:
    json.dump(out, fh)
print({k: len(v) for k, v in out.items() if isinstance(v, list)})
