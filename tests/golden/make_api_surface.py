"""Generate tests/golden/reference_api_surface.json: the public Python surface of the reference package (nrontsis/PILCO)
-- every module-level function, every class and, per class, every method with its positional parameter names -- read
from its sources with ``ast`` (never imported or executed).  tests/test_api_surface.py checks this package against it.

    python tests/golden/make_api_surface.py <path to a checkout of the reference>
"""
import ast
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
MODULES = {
    "pilco/models/mgpr.py": "pilco.models.mgpr",
    "pilco/models/smgpr.py": "pilco.models.smgpr",
    "pilco/models/pilco.py": "pilco.models.pilco",
    "pilco/controllers.py": "pilco.controllers",
    "pilco/rewards.py": "pilco.rewards",
    "safe_pilco_extension/rewards_safe.py": "safe_pilco_extension.rewards_safe",
    "safe_pilco_extension/safe_pilco.py": "safe_pilco_extension.safe_pilco",
}


def surface(ref_root):
    out = {}
    for path, modname in MODULES.items():
        tree = ast.parse(open(os.path.join(ref_root, path)).read())
        mod = {"functions": [], "classes": {}}
        for node in tree.body:
            if isinstance(node, ast.FunctionDef):
                mod["functions"].append(node.name)
            elif isinstance(node, ast.ClassDef):
                mod["classes"][node.name] = {item.name: [a.arg for a in item.args.args]
                                             for item in node.body if isinstance(item, ast.FunctionDef)}
        out[modname] = mod
    return out


if __name__ == "__main__":
    with open(os.path.join(HERE, "reference_api_surface.json"), "w") as f:
        json.dump(surface(sys.argv[1]), f, indent=1, sort_keys=True)
        f.write("\n")
