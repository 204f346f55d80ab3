"""Generates tests/golden/scan_orders.json: the Hilbert and zigzag patch orders as the reference's own functions
(_d2xy, hilbert_indices, zigzag_indices in flaxdiff/models/hilbert.py) compute them.  jax need not be installed: the
three functions are lifted out of the source with `ast` and run with numpy standing in for jax.numpy.
    python tests/golden/make_scan_order_fixture.py <flaxdiff checkout>
"""
import ast
import json
import math
import os
import sys

import numpy as np

GRIDS = [(1, 1), (2, 2), (4, 4), (8, 8), (16, 16), (64, 64), (6, 4), (3, 5), (16, 8)]

src = open(os.path.join(sys.argv[1], "flaxdiff", "models", "hilbert.py")).read()
tree = ast.parse(src)
wanted = {"_d2xy", "hilbert_indices", "zigzag_indices"}
mod = ast.Module(body=[n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in wanted], type_ignores=[])
ns = {"jnp": np, "np": np, "math": math, "Tuple": tuple}
exec(compile(mod, "hilbert.py", "exec"), ns)
out = {}
for HP, WP in GRIDS:
    out[f"{HP}x{WP}"] = {"hilbert": [int(v) for v in ns["hilbert_indices"](HP, WP)],
                         "zigzag": [int(v) for v in ns["zigzag_indices"](HP, WP)]}
json.dump(out, open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "scan_orders.json"), "w"))
print({k: len(v["hilbert"]) for k, v in out.items()})
