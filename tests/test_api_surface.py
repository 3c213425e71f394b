"""Drop-in check of the Python boundary (SURVEY.md section 8b-i): every class, method, property and module-level function
the reference defines in pilco/ and safe_pilco_extension/ must exist here under the same import path with the same
leading positional parameters.  The reference's surface is stored in tests/golden/reference_api_surface.json
(tests/golden/make_api_surface.py extracts it from the reference's sources with ``ast``)."""
import importlib
import inspect
import json
import os

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_api_surface.json")


def test_public_surface_matches_reference():
    import pilco  # noqa: F401  (installs the alias modules)
    checked, problems = 0, []
    for modname, ref in json.load(open(GOLDEN)).items():
        mod = importlib.import_module(modname)
        for name in ref["functions"]:
            checked += 1
            if not hasattr(mod, name):
                problems.append("missing function %s.%s" % (modname, name))
        for cname, methods in ref["classes"].items():
            cls = getattr(mod, cname, None)
            if cls is None:
                problems.append("missing class %s.%s" % (modname, cname))
                continue
            for mname, ref_args in methods.items():
                checked += 1
                if not hasattr(cls, mname):
                    problems.append("missing %s.%s.%s" % (modname, cname, mname))
                    continue
                static = inspect.getattr_static(cls, mname)
                if isinstance(static, property):
                    continue
                our_args = list(inspect.signature(getattr(cls, mname)).parameters)
                if our_args[:len(ref_args)] != ref_args:
                    problems.append("signature %s.%s.%s: reference %s, here %s" % (modname, cname, mname, ref_args, our_args))
    assert not problems, "\n".join(problems)
    assert checked >= 50
