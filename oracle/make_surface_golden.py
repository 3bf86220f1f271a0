"""Generate tests/golden/reference_surface.json: the plugin surface of ray_lightning (constructor and method
signatures, ``_RayOutput`` fields, module-level names), read by AST from a checkout of its sources — it cannot be
imported without ray / pytorch_lightning.  tests/test_surface_conformance.py compares this package against it.

    python -m oracle.make_surface_golden /path/to/ray_lightning-checkout
"""
import ast
import json
import os
import sys

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "reference_surface.json")


def _parse(ref, path):
    with open(os.path.join(ref, path)) as f:
        return ast.parse(f.read())


def _cls(ref, path, name):
    for node in ast.walk(_parse(ref, path)):
        if isinstance(node, ast.ClassDef) and node.name == name:
            return node
    raise KeyError(name)


def _sig(fn):
    """(positional (name, default) pairs, *args name, **kwargs name, keyword-only names); a default that is not a
    literal is recorded as "<expr>"."""
    a = fn.args
    names = [x.arg for x in a.args]
    defaults = [None] * (len(names) - len(a.defaults)) + [ast.literal_eval(d) if isinstance(d, ast.Constant) else "<expr>" for d in a.defaults]
    return [list(zip(names, defaults)), a.vararg.arg if a.vararg else None, a.kwarg.arg if a.kwarg else None,
            [k.arg for k in a.kwonlyargs]]


def _methods(node):
    return {n.name: _sig(n) for n in node.body if isinstance(n, ast.FunctionDef)}


def surface(root):
    ref = os.path.join(root, "ray_lightning")
    init = _parse(ref, "__init__.py")
    out = _cls(ref, "launchers/utils.py", "_RayOutput")

    def top_level(path):
        return sorted(n.name for n in _parse(ref, path).body if isinstance(n, (ast.FunctionDef, ast.ClassDef)))

    return {
        "RayStrategy": _methods(_cls(ref, "ray_ddp.py", "RayStrategy")),
        "HorovodRayStrategy": _methods(_cls(ref, "ray_horovod.py", "HorovodRayStrategy")),
        "RayLauncher": _methods(_cls(ref, "launchers/ray_launcher.py", "RayLauncher")),
        "RayExecutor": _methods(_cls(ref, "launchers/utils.py", "RayExecutor")),
        "RayHorovodLauncher": _methods(_cls(ref, "launchers/ray_horovod_launcher.py", "RayHorovodLauncher")),
        "_RayOutput_fields": [n.target.id for n in out.body if isinstance(n, ast.AnnAssign)],
        "__all__": next(ast.literal_eval(n.value) for n in init.body if isinstance(n, ast.Assign) and n.targets[0].id == "__all__"),
        "session_names": top_level("session.py"),
        "util_names": top_level("util.py"),
    }


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    with open(GOLDEN, "w") as f:
        json.dump(surface(sys.argv[1]), f, sort_keys=True, separators=(",", ":"))
        f.write("\n")
    print(GOLDEN)
