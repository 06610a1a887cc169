"""Every entry point of liblmod_b200.so is launched from one place: a call(...) in llavamod/kernels.py.  A second launch site with its
own hand-copied argument list can drift from the first (a swapped stride, a dropped flag) without any test of the other site noticing."""
import ast
import os
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "llava-mod_b200", "llavamod")


def call_sites():
    """-> [(module path relative to the package, [lmod_* names in the first argument])] for every call(...) / X.call(...) in llavamod/."""
    sites = []
    for d, _, files in os.walk(PKG):
        for f in sorted(files):
            if not f.endswith(".py"):
                continue
            path = os.path.join(d, f)
            with open(path) as fh:
                tree = ast.parse(fh.read(), path)
            for node in ast.walk(tree):
                if not isinstance(node, ast.Call):
                    continue
                fn = node.func
                if not ((isinstance(fn, ast.Name) and fn.id == "call") or (isinstance(fn, ast.Attribute) and fn.attr == "call")):
                    continue
                names = [c.value for c in ast.walk(node.args[0]) if isinstance(c, ast.Constant) and isinstance(c.value, str)
                         and c.value.startswith("lmod_")] if node.args else []
                sites.append((os.path.relpath(path, PKG), names))
    return sites


def test_every_entry_point_has_one_launch_site():
    sites = call_sites()
    assert len(sites) >= 40
    counts = Counter(n for _, names in sites for n in names)
    assert {n: c for n, c in counts.items() if c > 1} == {}


def test_only_kernels_py_launches():
    assert sorted({m for m, _ in call_sites()} - {"kernels.py"}) == []
