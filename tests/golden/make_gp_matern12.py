"""Generates tests/golden/gp_matern12.npz: oracle/make_golden.py's gen_gp on a Matern-1/2 model whose training set
repeats rows.

    python tests/golden/make_gp_matern12.py

Reduced config: Ackley in 5 dimensions, n = 112 of which the last 12 rows repeat the first 12 (r^2 = 0 pairs), 256
candidates, q = 4, seed 1240.
Test infrastructure; never imported by hebo_b200/.
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gp_oracle as O          # noqa: E402
from oracle import make_golden             # noqa: E402

REPEATS = 12


def main():
    problem = O.synthetic_problem

    def with_repeats(cfg, n, d, seed):
        X, y = problem(cfg, n, d, seed)
        X[n - REPEATS:] = X[:REPEATS]
        return X, y
    O.synthetic_problem = with_repeats
    try:
        make_golden.gen_gp("matern12", "ackley", 112, 5, 256, 4, "matern12", 1240)
    finally:
        O.synthetic_problem = problem
    print("wrote", os.path.join(make_golden.OUT, "gp_matern12.npz"))


if __name__ == "__main__":
    main()
