"""Sensors.  ``Lidar.measure`` is one launch of the ray-cast kernel (ref vmas/simulator/sensors.py)."""
from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Callable, Tuple, Union

import torch

from .utils import Color

_NO_RENDERING = "Rendering is outside the scope of the CUDA hot-path build"


class Sensor(ABC):
    """Something mounted on an agent that is read with ``measure()`` (ref sensors.py:21-44).
    ``agent`` is filled in by ``Agent.__init__`` when the sensor is handed to it."""

    def __init__(self, world):
        super().__init__()
        self._world = world
        self.agent = None

    @abstractmethod
    def measure(self):
        raise NotImplementedError

    def to(self, device: torch.device):
        raise NotImplementedError

    def render(self, env_index: int = 0):
        raise NotImplementedError(_NO_RENDERING)


class Lidar(Sensor):
    """``n_rays`` equally spaced rays in the agent's frame (ref sensors.py:47-123).

    A full-circle sweep drops the duplicated end angle (ref sensors.py:61-68).  ``measure``
    returns ``[B, n_rays]`` ranges, ``max_range`` where nothing is hit.
    """

    def __init__(
        self,
        world,
        angle_start: float = 0.0,
        angle_end: float = 2 * torch.pi,
        n_rays: int = 8,
        max_range: float = 1.0,
        entity_filter: Callable = lambda _: True,
        render_color: Union[Color, Tuple[float, float, float]] = Color.GRAY,
        alpha: float = 1.0,
        render: bool = True,
    ):
        super().__init__(world)
        closes_the_circle = (angle_start - angle_end) % (torch.pi * 2) < 1e-5
        n_points = n_rays + 1 if closes_the_circle else n_rays
        sweep = torch.linspace(angle_start, angle_end, n_points, device=world.device)[:n_rays]
        self._angles = sweep.repeat(world.batch_dim, 1)  # [B, n_rays], agent frame
        self._max_range = max_range
        self._entity_filter = entity_filter
        self._last_measurement = None
        # rendering options are carried for API compatibility only
        self._render, self._render_color, self._alpha = render, render_color, alpha

    def measure(self, vectorized: bool = True):
        # ``vectorized`` is accepted for API compatibility: both values run the same kernel
        # (the reference's per-ray python loop, sensors.py:102-113, has no counterpart here).
        self._last_measurement = self._world._get_backend().lidar_measure(self)
        return self._last_measurement

    @property
    def entity_filter(self):
        return self._entity_filter

    @entity_filter.setter
    def entity_filter(self, entity_filter: Callable):
        self._entity_filter = entity_filter
        if self._world is not None:  # the set of entities the rays can hit is part of the compiled plan
            self._world._invalidate_plan()

    def to(self, device: torch.device):
        self._angles = self._angles.to(device)

    # -- rendering attributes (kept so scenario files that read them still load) -------------------
    @property
    def render_color(self):
        colour = self._render_color
        return colour.value if isinstance(colour, Color) else colour

    @property
    def alpha(self):
        return self._alpha

    def set_render(self, render: bool):
        self._render = render
