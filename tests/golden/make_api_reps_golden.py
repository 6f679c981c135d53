"""Generate tests/golden/reference_api_reps.json: the constructor signature, public members, bases and logged tabular keys
of the reference's REPS, extracted from the reference SOURCE with `ast` by the helpers of make_api_golden.py (nothing is
imported).

Run:  python tests/golden/make_api_reps_golden.py     (needs the reference tree; the tests only read the committed JSON)
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_api_golden import REF, describe, tabular_keys  # noqa: E402

OUT = os.path.join(HERE, "reference_api_reps.json")
REL = "rllab/algos/reps.py"


def main():
    tree = ast.parse(open(os.path.join(REF, REL)).read())
    api = {}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == "REPS":
            d = describe(node)
            d["mirror"] = "rllab_b200.algos.reps.REPS"
            d["reference_file"] = REL
            d["bases"] = [ast.unparse(b) for b in node.bases]
            d["tabular"] = tabular_keys(node)
            api["REPS"] = d
    assert "REPS" in api
    with open(OUT, "w") as f:
        json.dump(api, f, indent=1, sort_keys=True, default=str)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
