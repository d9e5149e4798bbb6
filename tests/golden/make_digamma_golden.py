"""Generates tests/golden/digamma_golden.json with mpmath (50 digits).

Boost.Math (the reference's digamma, CollapsedEMOptimizer.cpp:119,127,256,269) is not
vendored in the salmon source tree, so the pin for the oracle's restatement is the function
itself: high-precision values at seeded points covering every branch (recurrence
up/down, the [1,2] rational, the x>=10 asymptotic series, the root neighbourhood).
Run: python tests/golden/make_digamma_golden.py
"""
import json
import os
import random

import mpmath

mpmath.mp.dps = 50
random.seed(20260922)
xs = [1.0000000001e-10, 1e-9, 1e-6, 1e-3, 1e-2, 0.1, 0.5, 0.99, 1.0, 1.25, 1.4616321449683623, 1.5,
      1.999, 2.0, 2.5, 3.7, 9.999, 10.0, 10.5, 50.0, 100.0, 1e4, 2.0407426e7, 1e9, 1e12]
xs += [10 ** random.uniform(-9.9, 9) for _ in range(400)]
rows = []
for x in xs:
    v = mpmath.digamma(mpmath.mpf(x))
    rows.append({"x": float(x).hex(), "digamma": mpmath.nstr(v, 25)})
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "digamma_golden.json")
with open(out, "w") as f:
    json.dump({"source": "mpmath %s, mp.dps=50" % mpmath.__version__, "rows": rows}, f, indent=0)
print("wrote", out, len(rows))
