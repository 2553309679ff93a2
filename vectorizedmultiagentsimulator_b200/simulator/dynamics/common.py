"""Base class of the action→force models.

A ``Dynamics`` object is owned by exactly one agent.  Right before ``World.step`` the environment
calls :meth:`check_and_process_action`, which turns ``agent.action.u`` into ``agent.state.force`` /
``agent.state.torque`` (behavioural contract of ref vmas/simulator/dynamics/common.py:12-53).
"""
from __future__ import annotations

import abc
from typing import Optional


class Dynamics(abc.ABC):
    """Maps an agent's processed action ``u`` to the force and torque the physics step applies."""

    _UNBOUND = (
        "You need to add the dynamics to an agent during construction before accessing its properties"
    )

    def __init__(self):
        self._agent: Optional[object] = None

    # -- ownership --------------------------------------------------------------------------
    def _get_agent(self):
        owner = self._agent
        if owner is None:
            raise ValueError(self._UNBOUND)
        return owner

    def _set_agent(self, owner):
        if self._agent is not None:
            raise ValueError("Agent in dynamics has already been set")
        self._agent = owner

    agent = property(_get_agent, _set_agent, doc="The agent this model drives (set once by ``Agent``).")

    # -- lifecycle hooks (stateful models override) ---------------------------------------------
    def reset(self, index=None):
        """Called on ``world.reset(index)``; stateless models have nothing to do."""

    def zero_grad(self):
        """Kept for API compatibility; the CUDA path carries no autograd graph."""

    # -- the contract ---------------------------------------------------------------------------
    @property
    @abc.abstractmethod
    def needed_action_size(self) -> int:
        """How many leading components of ``agent.action.u`` this model consumes."""

    @abc.abstractmethod
    def process_action(self):
        """Write ``agent.state.force`` / ``agent.state.torque`` from ``agent.action.u``."""

    def check_and_process_action(self):
        provided = self.agent.action.u.shape[1]
        required = self.needed_action_size
        if provided < required:
            raise ValueError(
                f"Agent action size {provided} is less than the required dynamics action size {required}"
            )
        self.process_action()
