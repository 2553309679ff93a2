"""Scenario lookup by file name (ref vmas/scenarios/__init__.py:11-24).

Search order: this directory (the scenarios re-written for the CUDA build), then every
directory listed in ``$VMAS_SCENARIO_PATH`` (``os.pathsep``-separated; walked recursively), so
an unmodified reference checkout's scenario files can be dropped in.  Files from outside this
package import ``vmas.simulator...``; :func:`..compat.install_vmas_alias` is called so those
imports resolve to this package.
"""
import importlib
import importlib.util
import os
from pathlib import Path


def _find(name: str):
    if os.path.isfile(name):
        return name
    roots = [os.path.dirname(__file__)]
    roots += [p for p in os.environ.get("VMAS_SCENARIO_PATH", "").split(os.pathsep) if p]
    for root in roots:
        for dirpath, _, filenames in os.walk(root):
            for filename in filenames:
                if filename == "__init__.py":
                    continue
                if name == filename or Path(name) == Path(dirpath) / Path(filename):
                    return os.path.join(dirpath, filename)
    return None


def load(name: str):
    pathname = _find(name)
    assert pathname is not None, f"{name} scenario not found."
    here = os.path.dirname(os.path.abspath(__file__))
    if os.path.abspath(pathname).startswith(here + os.sep):
        # one of this package's scenarios: a regular submodule (they use relative imports)
        rel = os.path.relpath(os.path.abspath(pathname), here)[: -len(".py")]
        return importlib.import_module(__name__ + "." + rel.replace(os.sep, "."))
    from ..compat import install_vmas_alias

    install_vmas_alias()
    spec = importlib.util.spec_from_file_location("", pathname)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module
