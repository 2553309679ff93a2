"""``make_env``: scenario name (or instance) → ``Environment`` (ref vmas/make_env.py:14-101)."""
from __future__ import annotations

from typing import Optional, Union

import torch

from . import scenarios
from .simulator.environment import Environment, Wrapper
from .simulator.environment.environment import check_obs_dtype
from .simulator.scenario import BaseScenario
from .simulator.utils import DEVICE_TYPING


def make_env(
    scenario: Union[str, BaseScenario],
    num_envs: int,
    device: DEVICE_TYPING = "cuda",
    continuous_actions: bool = True,
    wrapper: Optional[Union[Wrapper, str]] = None,
    max_steps: Optional[int] = None,
    seed: Optional[int] = None,
    dict_spaces: bool = False,
    multidiscrete_actions: bool = False,
    clamp_actions: bool = False,
    grad_enabled: bool = False,
    terminated_truncated: bool = False,
    wrapper_kwargs: Optional[dict] = None,
    cuda_graph: bool = False,
    action_checks: Optional[str] = None,
    auto_reset: bool = False,
    obs_dtype: torch.dtype = torch.float32,
    **kwargs,
):
    """Create a vectorised environment.

    Arguments are the reference's.  ``scenario`` may be a scenario file name (looked up first
    among this package's scenarios, then in ``$VMAS_SCENARIO_PATH`` directories — e.g. an
    unmodified reference checkout's ``vmas/scenarios``), a path to a scenario file, or a
    ``BaseScenario`` instance.  ``device`` defaults to ``"cuda"``: the physics only runs there.
    ``cuda_graph=True`` replays one captured CUDA graph per ``step`` (graph-safe scenarios only),
    ``action_checks`` selects ``"sync"`` / ``"deferred"`` / ``"off"`` validation of the input
    actions, ``auto_reset=True`` resets finished envs on the device inside ``step`` (see
    ``Environment``), ``obs_dtype`` (``torch.float32``, ``torch.float16`` or ``torch.bfloat16``) is the type
    every fp32 observation leaf is handed out as.  Remaining ``kwargs`` go to ``Scenario.make_world``.
    """
    check_obs_dtype(obs_dtype)
    if wrapper is not None and obs_dtype == torch.bfloat16:
        raise ValueError("obs_dtype=torch.bfloat16 cannot be combined with a wrapper: the adapters convert "
                         "observations to numpy, which has no bfloat16 (torch.float16 works)")
    env = Environment(
        _as_scenario(scenario),
        num_envs=num_envs,
        device=device,
        max_steps=max_steps,
        seed=seed,
        # how actions are read and outputs are laid out
        continuous_actions=continuous_actions,
        multidiscrete_actions=multidiscrete_actions,
        clamp_actions=clamp_actions,
        dict_spaces=dict_spaces,
        terminated_truncated=terminated_truncated,
        grad_enabled=grad_enabled,
        # additions of this package
        cuda_graph=cuda_graph,
        action_checks=action_checks,
        auto_reset=auto_reset,
        obs_dtype=obs_dtype,
        **kwargs,
    )
    if wrapper is None:
        return env
    adapter = Wrapper[wrapper.upper()] if isinstance(wrapper, str) else wrapper
    return adapter.get_env(env, **(wrapper_kwargs or {}))


def _as_scenario(scenario: Union[str, BaseScenario]) -> BaseScenario:
    """A ``BaseScenario`` instance from a name, a file path or an instance."""
    if isinstance(scenario, BaseScenario):
        return scenario
    file_name = scenario if scenario.endswith(".py") else scenario + ".py"
    return scenarios.load(file_name).Scenario()
