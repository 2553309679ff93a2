"""Drop-in import alias: makes ``import vmas...`` resolve to this package.

Existing scenario files start with lines such as ``from vmas.simulator.core import Agent, Box,
Landmark, Line, Sphere, World`` (e.g. reference scenarios/balance.py:9).  ``install_vmas_alias``
registers this package's modules under the ``vmas`` names so those files load unchanged.
It refuses to shadow a real ``vmas`` installation that is already imported.
"""
from __future__ import annotations

import importlib
import sys
import types

_PKG = __name__.rsplit(".", 1)[0]

_MODULES = [
    "simulator",
    "simulator.core",
    "simulator.utils",
    "simulator.scenario",
    "simulator.sensors",
    "simulator.joints",
    "simulator.dynamics",
    "simulator.dynamics.common",
    "simulator.dynamics.basic",
    "simulator.dynamics.holonomic",
    "simulator.dynamics.holonomic_with_rot",
    "simulator.dynamics.forward",
    "simulator.dynamics.roatation",
    "simulator.dynamics.static",
    "simulator.dynamics.diff_drive",
    "simulator.dynamics.kinematic_bicycle",
    "simulator.dynamics.drone",
    "simulator.controllers",
    "simulator.controllers.velocity_controller",
    "simulator.environment",
    "simulator.environment.environment",
    "simulator.heuristic_policy",
    "make_env",
    "scenarios",
]


def _render_interactively(*args, **kwargs):
    raise NotImplementedError("Interactive rendering is outside the scope of the CUDA hot-path build")


def install_vmas_alias(force: bool = False) -> None:
    existing = sys.modules.get("vmas")
    if existing is not None:
        if getattr(existing, "__vmas_b200_alias__", False):
            return
        if not force:
            raise RuntimeError(
                "A different 'vmas' package is already imported; refusing to alias over it "
                "(pass force=True to override)"
            )
    root = importlib.import_module(_PKG)
    alias = types.ModuleType("vmas")
    alias.__dict__.update(
        {k: v for k, v in root.__dict__.items() if not k.startswith("__")}
    )
    alias.__path__ = []  # mark as package
    alias.__vmas_b200_alias__ = True
    alias.render_interactively = _render_interactively
    sys.modules["vmas"] = alias
    for name in _MODULES:
        try:
            mod = importlib.import_module(f"{_PKG}.{name}")
        except ModuleNotFoundError:
            continue
        sys.modules[f"vmas.{name}"] = mod
        parent, _, leaf = name.rpartition(".")
        holder = sys.modules["vmas" + ("." + parent if parent else "")]
        setattr(holder, leaf, mod)
