"""Generate tests/golden/reference_api_vf.json: constructor signatures, public members and tabular keys of the reference
classes behind GaussianMLPBaseline, extracted from the reference SOURCE with `ast` by the helpers of
make_api_golden.py (nothing is imported).

Run:  python tests/golden/make_api_vf_golden.py     (needs the reference tree; the tests only read the committed JSON)
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_api_golden import REF, describe, tabular_keys  # noqa: E402

OUT = os.path.join(HERE, "reference_api_vf.json")
CLASSES = {
    "rllab/baselines/gaussian_mlp_baseline.py": {
        "GaussianMLPBaseline": "rllab_b200.baselines.gaussian_mlp_baseline.GaussianMLPBaseline"},
    "rllab/regressors/gaussian_mlp_regressor.py": {
        "GaussianMLPRegressor": "rllab_b200.regressors.gaussian_mlp_regressor.GaussianMLPRegressor"},
    "rllab/optimizers/penalty_lbfgs_optimizer.py": {
        "PenaltyLbfgsOptimizer": "rllab_b200.optimizers.penalty_lbfgs_optimizer.PenaltyLbfgsOptimizer"},
    "rllab/optimizers/lbfgs_optimizer.py": {"LbfgsOptimizer": "rllab_b200.optimizers.lbfgs_optimizer.LbfgsOptimizer"},
}
def prefixed_tabular_keys(tree):
    """record_tabular(prefix + 'Key', ...) calls: the 'Key' suffixes (the regressor prefixes its name + '_')."""
    keys = []
    for n in ast.walk(tree):
        if (isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and n.func.attr == "record_tabular" and n.args
                and isinstance(n.args[0], ast.BinOp) and isinstance(n.args[0].right, ast.Constant)
                and n.args[0].right.value not in keys):
            keys.append(n.args[0].right.value)
    return keys


TABULAR = {"rllab/regressors/gaussian_mlp_regressor.py": ["rllab_b200/regressors/gaussian_mlp_regressor.py"]}


def main():
    api = {}
    for rel, classes in CLASSES.items():
        tree = ast.parse(open(os.path.join(REF, rel)).read())
        for node in tree.body:
            if isinstance(node, ast.ClassDef) and node.name in classes:
                d = describe(node)
                d["mirror"] = classes[node.name]
                d["reference_file"] = rel
                api[node.name] = d
    missing = {c for cl in CLASSES.values() for c in cl} - set(api)
    assert not missing, missing
    api["__tabular__"] = {}
    for rel, mirrors in TABULAR.items():
        tree = ast.parse(open(os.path.join(REF, rel)).read())
        api["__tabular__"][rel] = {"keys": tabular_keys(tree), "prefixed_keys": prefixed_tabular_keys(tree),
                                   "mirrors": mirrors}
    with open(OUT, "w") as f:
        json.dump(api, f, indent=1, sort_keys=True, default=str)
    print("wrote", OUT, len(api) - 1, "classes")


if __name__ == "__main__":
    main()
