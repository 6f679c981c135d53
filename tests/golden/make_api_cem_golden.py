"""Generate tests/golden/reference_api_cem.json: the constructor signature and public members of the reference's CEM,
extracted from the reference SOURCE with `ast` by the helpers of make_api_golden.py (nothing is imported).

Run:  python tests/golden/make_api_cem_golden.py     (needs the reference tree; the tests only read the committed JSON)
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_api_golden import REF, describe  # noqa: E402

OUT = os.path.join(HERE, "reference_api_cem.json")
CLASSES = {
    "rllab/algos/cem.py": {"CEM": "rllab_b200.algos.cem.CEM"},
}


def main():
    api = {}
    for rel, classes in CLASSES.items():
        tree = ast.parse(open(os.path.join(REF, rel)).read())
        for node in tree.body:
            if isinstance(node, ast.ClassDef) and node.name in classes:
                d = describe(node)
                d["mirror"] = classes[node.name]
                d["reference_file"] = rel
                d["bases"] = [ast.unparse(b) for b in node.bases]
                api[node.name] = d
    missing = {c for cl in CLASSES.values() for c in cl} - set(api)
    assert not missing, missing
    with open(OUT, "w") as f:
        json.dump(api, f, indent=1, sort_keys=True, default=str)
    print("wrote", OUT, len(api), "classes")


if __name__ == "__main__":
    main()
