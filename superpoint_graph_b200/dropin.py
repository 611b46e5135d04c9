"""Installs the sm_90a operators under the reference's module names.

The reference's trainer does `from learning import spg, graphnet, pointnet, metrics` and
`import ecc`-style imports (ref: learning/main.py:31-37, learning/spg.py:21, learning/modules.py:14,
learning/ecc/utils.py:15).  `install()` registers this package's mirrors in `sys.modules` *before*
those imports run, so `learning/main.py` itself stays untouched:

    learning.pointnet  -> superpoint_graph_b200.spg_pointnet
    learning.graphnet  -> superpoint_graph_b200.spg_graphnet
    learning.modules   -> superpoint_graph_b200.spg_modules
    learning.ecc, ecc  -> superpoint_graph_b200.spg_ecc

Everything else of `learning/` (dataset adapters, spg.py loader, metrics, main.py) keeps coming from
the reference checkout given by `reference_root`.
"""
import importlib
import os
import sys
import types

_MIRRORS = {
    "pointnet": "spg_pointnet",
    "graphnet": "spg_graphnet",
    "modules": "spg_modules",
    "ecc": "spg_ecc",
}


def install(reference_root=None):
    """Registers the mirrors; returns the `learning` package object."""
    pkg = sys.modules.get("learning")
    if pkg is None:
        pkg = types.ModuleType("learning")
        pkg.__path__ = []
        sys.modules["learning"] = pkg
    if reference_root is not None:
        learning_dir = os.path.join(reference_root, "learning")
        if learning_dir not in pkg.__path__:
            pkg.__path__.append(learning_dir)  # dataset adapters, spg.py, metrics.py, main.py
        if reference_root not in sys.path:
            sys.path.insert(0, reference_root)
    for ref_name, ours in _MIRRORS.items():
        mod = importlib.import_module("superpoint_graph_b200." + ours)
        sys.modules["learning." + ref_name] = mod
        setattr(pkg, ref_name, mod)
    sys.modules["ecc"] = sys.modules["learning.ecc"]  # bare `import ecc` (ecc/utils.py:15)
    return pkg


def uninstall():
    for ref_name in _MIRRORS:
        sys.modules.pop("learning." + ref_name, None)
    sys.modules.pop("ecc", None)
