"""Host-side object model: shapes, entities, agents and the ``World``.

This module keeps the class surface scenarios program against in the reference
(``from vmas.simulator.core import Agent, Box, Landmark, Line, Sphere, World``; reference
``vmas/simulator/core.py``) but inverts data ownership and removes all physics from
Python:

* state lives in a contiguous :class:`~.slab.StateSlab`; ``entity.state.pos`` & co. are
  writable views into it, and their setters copy *into* the slab;
* ``World.step`` / ``cast_rays`` / ``get_distance`` / ``is_overlapping`` are single calls
  into the sm_90a kernels through the C-ABI library (``include/vmas_b200.h``).  There is no
  torch-eager or CPU implementation of the physics in this package: on a non-CUDA device, or
  without the built library, those calls raise.

Reference behaviour each piece stands in for is cited inline as ``ref core.py:<lines>``.
"""
from __future__ import annotations

import math
import os
from abc import ABC, abstractmethod
from typing import Callable, List, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor

from .dynamics.common import Dynamics
from .dynamics.holonomic import Holonomic
from .slab import StateSlab
from .utils import (
    ANGULAR_FRICTION,
    COLLISION_FORCE,
    Color,
    DRAG,
    JOINT_FORCE,
    LINEAR_FRICTION,
    Observable,
    TORQUE_CONSTRAINT_FORCE,
    X,
    Y,
)


class TorchVectorizedObject:
    """Anything that carries a leading ``batch_dim`` and lives on one device (ref core.py:48-82)."""

    def __init__(self, batch_dim: int = None, device: torch.device = None):
        self._batch_dim = batch_dim
        self._device = device

    @property
    def batch_dim(self):
        return self._batch_dim

    @batch_dim.setter
    def batch_dim(self, batch_dim: int):
        assert self._batch_dim is None, "You can set batch dim only once"
        self._batch_dim = batch_dim

    @property
    def device(self):
        return self._device

    @device.setter
    def device(self, device: torch.device):
        self._device = device

    def _check_batch_index(self, batch_index):
        if batch_index is not None and isinstance(batch_index, int):
            assert (
                0 <= batch_index < self.batch_dim
            ), f"Index must be between 0 and {self.batch_dim}, got {batch_index}"

    def to(self, device: torch.device):
        self.device = device
        for attr, value in self.__dict__.items():
            if isinstance(value, Tensor):
                self.__dict__[attr] = value.to(device)


# ----------------------------------------------------------------------------------------
# Shapes (ref core.py:85-203)
# ----------------------------------------------------------------------------------------
class Shape(ABC):
    @abstractmethod
    def moment_of_inertia(self, mass: float):
        raise NotImplementedError

    @abstractmethod
    def get_delta_from_anchor(self, anchor: Tuple[float, float]) -> Tuple[float, float]:
        raise NotImplementedError

    @abstractmethod
    def circumscribed_radius(self):
        raise NotImplementedError

    def get_geometry(self):
        raise NotImplementedError("Rendering is outside the scope of the CUDA hot-path build")


class Box(Shape):
    def __init__(self, length: float = 0.3, width: float = 0.1, hollow: bool = False):
        assert length > 0, f"Length must be > 0, got {length}"
        assert width > 0, f"Width must be > 0, got {length}"
        self._length = length
        self._width = width
        self.hollow = hollow

    @property
    def length(self):
        return self._length

    @property
    def width(self):
        return self._width

    def get_delta_from_anchor(self, anchor):
        return anchor[X] * self.length / 2, anchor[Y] * self.width / 2

    def moment_of_inertia(self, mass: float):
        return (1 / 12) * mass * (self.length**2 + self.width**2)

    def circumscribed_radius(self):
        return math.sqrt((self.length / 2) ** 2 + (self.width / 2) ** 2)


class Sphere(Shape):
    def __init__(self, radius: float = 0.05):
        assert radius > 0, f"Radius must be > 0, got {radius}"
        self._radius = radius

    @property
    def radius(self):
        return self._radius

    def get_delta_from_anchor(self, anchor):
        # fp32 on purpose, including the reference's "divide by norm*radius" rescale of
        # anchors outside the unit circle (ref core.py:151-158).
        delta = torch.tensor(
            [anchor[X] * self.radius, anchor[Y] * self.radius], dtype=torch.float32
        )
        norm = torch.linalg.vector_norm(delta)
        if norm > self.radius:
            delta = delta / (norm * self.radius)
        return tuple(delta.tolist())

    def moment_of_inertia(self, mass: float):
        return (1 / 2) * mass * self.radius**2

    def circumscribed_radius(self):
        return self.radius


class Line(Shape):
    def __init__(self, length: float = 0.5):
        assert length > 0, f"Length must be > 0, got {length}"
        self._length = length
        self._width = 2

    @property
    def length(self):
        return self._length

    @property
    def width(self):
        return self._width

    def moment_of_inertia(self, mass: float):
        return (1 / 12) * mass * (self.length**2)

    def circumscribed_radius(self):
        return self.length / 2

    def get_delta_from_anchor(self, anchor):
        return anchor[X] * self.length / 2, 0.0


def _zero_rows(t: Tensor, env_index) -> None:
    """``t[env_index] = 0`` for ``None`` (all rows), an int, or a ``[B]`` bool mask (no host sync)."""
    if env_index is None:
        t.zero_()
    elif isinstance(env_index, Tensor):
        t.masked_fill_(env_index.view(-1, *([1] * (t.dim() - 1))), 0.0)
    else:
        t[env_index] = 0.0


def _write_rows(dst: Tensor, new: Tensor, mask: Tensor) -> None:
    """``dst[mask] = new[mask]`` for a ``[B]`` bool mask without a host sync; ``new`` is a full
    ``[B, ...]`` tensor or broadcastable to one."""
    dst.copy_(torch.where(mask.view(-1, *([1] * (dst.dim() - 1))), new, dst))


# ----------------------------------------------------------------------------------------
# State containers (ref core.py:206-410).  Fields are views into the world's StateSlab
# once the entity has been packed; before that they are standalone [B, k] tensors.
# ----------------------------------------------------------------------------------------
_DEBUG_STATE_ALIASING = os.environ.get("VMAS_B200_DEBUG_STATE_ALIASING", "0") == "1"


class _SlabFields(TorchVectorizedObject):
    _NAMES: Tuple[str, ...] = ()

    def __init__(self):
        super().__init__()
        self._fields = {}

    def _get(self, name):
        value = self._fields.get(name)
        if _DEBUG_STATE_ALIASING and value is not None:
            # the reference hands out a tensor that the next step does not touch (it re-binds a new
            # one); here state is a view into the slab.  Debug aid for drop-in scenarios that keep raw
            # state tensors across a step without cloning (INTEGRATION.md): getters return copies.
            return value.clone()
        return value

    def _set(self, name, value: Tensor, same_shape_as: Optional[str] = None):
        assert (
            self._batch_dim is not None and self._device is not None
        ), "First add an entity to the world before setting its state"
        assert (
            value.shape[0] == self._batch_dim
        ), f"Internal state must match batch dim, got {value.shape[0]}, expected {self._batch_dim}"
        if same_shape_as is not None and self._fields.get(same_shape_as) is not None:
            other = self._fields[same_shape_as]
            assert (
                value.shape == other.shape
            ), f"{name} shape must match {same_shape_as} shape, got {value.shape} expected {other.shape}"
        cur = self._fields.get(name)
        if cur is None:
            self._fields[name] = value.to(self._device)
        else:
            assert cur.shape == value.shape, (
                f"Cannot re-shape state field '{name}' from {tuple(cur.shape)} to "
                f"{tuple(value.shape)}: it is a view into the world's state slab"
            )
            if value is not cur:
                cur.copy_(value)

    def _reset(self, env_index):
        for name in self._NAMES:
            t = self._fields.get(name)
            if t is not None:
                _zero_rows(t, env_index)

    def zero_grad(self):
        # The CUDA path is forward-only; nothing carries a graph.
        return

    def to(self, device: torch.device):
        self.device = device
        for name, t in list(self._fields.items()):
            if t is not None:
                self._fields[name] = t.to(device)


def _field(name, same_shape_as=None):
    def getter(self):
        return self._get(name)

    def setter(self, value):
        self._set(name, value, same_shape_as)

    return property(getter, setter)


class EntityState(_SlabFields):
    _NAMES = ("pos", "rot", "vel", "ang_vel")

    pos = _field("pos", same_shape_as="vel")
    vel = _field("vel", same_shape_as="pos")
    rot = _field("rot")
    ang_vel = _field("ang_vel")

    def _spawn(self, dim_c: int, dim_p: int):
        kw = dict(device=self.device, dtype=torch.float32)
        self.pos = torch.zeros(self.batch_dim, dim_p, **kw)
        self.vel = torch.zeros(self.batch_dim, dim_p, **kw)
        self.rot = torch.zeros(self.batch_dim, 1, **kw)
        self.ang_vel = torch.zeros(self.batch_dim, 1, **kw)


class AgentState(EntityState):
    _NAMES = ("c", "force", "torque") + EntityState._NAMES

    force = _field("force")
    torque = _field("torque")

    @property
    def c(self):
        return self._get("c")

    @c.setter
    def c(self, c: Tensor):
        assert (
            self._batch_dim is not None and self._device is not None
        ), "First add an entity to the world before setting its state"
        assert (
            c.shape[0] == self._batch_dim
        ), f"Internal state must match batch dim, got {c.shape[0]}, expected {self._batch_dim}"
        # communication state is not part of the physics slab: plain re-bind
        self._fields["c"] = c.to(self._device)

    def _spawn(self, dim_c: int, dim_p: int):
        kw = dict(device=self.device, dtype=torch.float32)
        if dim_c > 0:
            self.c = torch.zeros(self.batch_dim, dim_c, **kw)
        self.force = torch.zeros(self.batch_dim, dim_p, **kw)
        self.torque = torch.zeros(self.batch_dim, 1, **kw)
        super()._spawn(dim_c, dim_p)


class Action(TorchVectorizedObject):
    """Per-agent action buffers and their static ranges (ref core.py:414-534)."""

    def __init__(self, u_range, u_multiplier, u_noise, action_size: int):
        super().__init__()
        self._u_noise = u_noise
        self._u_range = u_range
        self._u_multiplier = u_multiplier
        self.action_size = action_size
        self._u = None
        self._c = None
        self._cache = {}
        for attr in (u_multiplier, u_range, u_noise):
            if isinstance(attr, List):
                assert len(attr) == action_size, (
                    "Action attributes u_... must be either a float or a list of floats"
                    " (one per action) all with same length"
                )

    def _checked(self, value: Tensor, what: str) -> Tensor:
        assert (
            self._batch_dim is not None and self._device is not None
        ), "First add an agent to the world before setting its action"
        assert (
            value.shape[0] == self._batch_dim
        ), f"{what} must match batch dim, got {value.shape[0]}, expected {self._batch_dim}"
        return value.to(self._device)

    @property
    def u(self):
        return self._u

    @u.setter
    def u(self, u: Tensor):
        self._u = self._checked(u, "Action")

    @property
    def c(self):
        return self._c

    @c.setter
    def c(self, c: Tensor):
        self._c = self._checked(c, "Action")

    @property
    def u_range(self):
        return self._u_range

    @property
    def u_multiplier(self):
        return self._u_multiplier

    @property
    def u_noise(self):
        return self._u_noise

    def _as_tensor(self, key, value):
        t = self._cache.get(key)
        dev = torch.device(self.device)
        if t is None or t.device.type != dev.type or (dev.index is not None and t.device.index != dev.index):
            t = torch.tensor(
                list(value) if isinstance(value, Sequence) else [value] * self.action_size,
                device=self.device,
                dtype=torch.float,
            )
            self._cache[key] = t
        return t

    @property
    def u_range_tensor(self):
        return self._as_tensor("range", self._u_range)

    @property
    def u_multiplier_tensor(self):
        return self._as_tensor("mult", self._u_multiplier)

    @property
    def u_noise_tensor(self):
        return self._as_tensor("noise", self._u_noise)

    def _reset(self, env_index):
        for name in ("_u", "_c"):
            t = getattr(self, name)
            if t is None:
                continue
            if env_index is None:
                setattr(self, name, torch.zeros_like(t))
            else:
                t = t.clone()
                _zero_rows(t, env_index)  # an int, or a [B] bool mask (no host sync)
                setattr(self, name, t)

    def zero_grad(self):
        return

    def to(self, device: torch.device):
        self.device = device
        self._cache.clear()
        for name in ("_u", "_c"):
            t = getattr(self, name)
            if t is not None:
                setattr(self, name, t.to(device))


#: physical parameters an entity may hold per env, as a [batch_dim, 1] fp32 tensor (domain randomisation)
PER_ENV_PARAMS = ("mass", "linear_friction", "angular_friction")


def _is_param_tensor(value) -> bool:
    return isinstance(value, Tensor) and value.dim() > 0


def _checked_param(entity_name: str, attr: str, value):
    """``value`` if it is a python number, None, a 0-d tensor or a 2-D ``[n, 1]`` fp32 tensor; else ValueError.
    (The batch size and the device are checked once the entity belongs to a world.)"""
    if value is None or isinstance(value, (int, float)) or not _is_param_tensor(value):
        return value
    if value.dtype != torch.float32 or value.dim() != 2 or value.shape[1] != 1:
        raise ValueError(
            f"Entity '{entity_name}': {attr} must be a python number or a float32 tensor of shape "
            f"[batch_dim, 1], got {value.dtype} {list(value.shape)}"
        )
    return value.detach().clone()


# ----------------------------------------------------------------------------------------
# Entities (ref core.py:538-1086)
# ----------------------------------------------------------------------------------------
class Entity(TorchVectorizedObject, Observable, ABC):
    def __init__(
        self,
        name: str,
        movable: bool = False,
        rotatable: bool = False,
        collide: bool = True,
        density: float = 25.0,
        mass: float = 1.0,
        shape: Shape = None,
        v_range: float = None,
        max_speed: float = None,
        color=Color.GRAY,
        is_joint: bool = False,
        drag: float = None,
        linear_friction: float = None,
        angular_friction: float = None,
        gravity: Union[float, Tensor] = None,
        collision_filter: Callable[["Entity"], bool] = lambda _: True,
    ):
        TorchVectorizedObject.__init__(self)
        Observable.__init__(self)
        self._name = name
        self._movable = movable
        self._rotatable = rotatable
        self._collide = collide
        self._density = density
        self._mass = _checked_param(name, "mass", mass)
        self._max_speed = max_speed
        self._v_range = v_range
        self._color = color
        self._shape = shape if shape is not None else Sphere()
        self._is_joint = is_joint
        self._collision_filter = collision_filter
        self._state = EntityState()
        self._drag = drag
        self._linear_friction = _checked_param(name, "linear_friction", linear_friction)
        self._angular_friction = _checked_param(name, "angular_friction", angular_friction)
        if gravity is None or isinstance(gravity, Tensor):
            self._gravity = gravity
        else:
            self._gravity = torch.tensor(gravity, dtype=torch.float32)
        self._goal = None
        self._render = None
        self._world = None  # set by World.add_*; used to invalidate the compiled plan

    # -- plan invalidation -------------------------------------------------------------
    def _touch(self):
        if self._world is not None:
            self._world._invalidate_plan()

    @TorchVectorizedObject.batch_dim.setter
    def batch_dim(self, batch_dim: int):
        TorchVectorizedObject.batch_dim.fset(self, batch_dim)
        self._state.batch_dim = batch_dim
        for attr in PER_ENV_PARAMS:  # a tensor given to the constructor meets its world's batch here
            value = getattr(self, "_" + attr)
            if _is_param_tensor(value) and batch_dim is not None and value.shape[0] != batch_dim:
                raise ValueError(
                    f"Entity '{self.name}': {attr} must be a float32 tensor of shape [batch_dim, 1] = "
                    f"[{batch_dim}, 1], got {list(value.shape)}"
                )

    def _set_param(self, attr: str, value):
        """Setter of a per-env-capable physical parameter (mass, linear / angular friction).

        A python number is structure, as before: the plan is rebuilt.  A ``[batch_dim, 1]`` fp32 tensor on the
        world's device is copied into a buffer the entity owns (allocated on the first tensor assignment and
        kept while the attribute stays a tensor), so a tensor after a tensor is data only: no plan rebuild and
        a captured CUDA graph keeps reading the same address."""
        value = _checked_param(self.name, attr, value)
        old = getattr(self, "_" + attr)
        if _is_param_tensor(value):
            if self.batch_dim is not None and value.shape[0] != self.batch_dim:
                raise ValueError(
                    f"Entity '{self.name}': {attr} must be a float32 tensor of shape [batch_dim, 1] = "
                    f"[{self.batch_dim}, 1], got {list(value.shape)}"
                )
            want = None if self.device is None else torch.device(self.device)
            if want is not None and (value.device.type != want.type or want.index not in (None, value.device.index)):
                raise ValueError(f"Entity '{self.name}': {attr} must be on the world's device {want}, got {value.device}")
            if _is_param_tensor(old) and old.shape == value.shape and old.device == value.device:
                if value.data_ptr() != old.data_ptr():
                    old.copy_(value)
                return
            setattr(self, "_" + attr, value.detach().clone())
        else:
            setattr(self, "_" + attr, value)
        self._touch()

    @property
    def is_rendering(self):
        if self._render is None:
            self.reset_render()
        return self._render

    def reset_render(self):
        self._render = torch.full((self.batch_dim,), True, device=self.device)

    def collides(self, entity: "Entity"):
        if not self.collide:
            return False
        return self._collision_filter(entity)

    # static physical attributes ----------------------------------------------------------
    @property
    def is_joint(self):
        return self._is_joint

    @property
    def mass(self):
        return self._mass

    @mass.setter
    def mass(self, mass):
        self._set_param("mass", mass)

    @property
    def moment_of_inertia(self):
        return self.shape.moment_of_inertia(self.mass)

    @property
    def state(self):
        return self._state

    @property
    def movable(self):
        return self._movable

    @property
    def collide(self):
        return self._collide

    @property
    def shape(self):
        return self._shape

    @property
    def max_speed(self):
        return self._max_speed

    @property
    def v_range(self):
        return self._v_range

    @property
    def name(self):
        return self._name

    @property
    def rotatable(self):
        return self._rotatable

    @property
    def color(self):
        if isinstance(self._color, Color):
            return self._color.value
        return self._color

    @color.setter
    def color(self, color):
        self._color = color

    @property
    def goal(self):
        return self._goal

    @goal.setter
    def goal(self, goal: "Entity"):
        self._goal = goal

    @property
    def drag(self):
        return self._drag

    @property
    def linear_friction(self):
        return self._linear_friction

    @linear_friction.setter
    def linear_friction(self, value):
        self._set_param("linear_friction", value)

    @property
    def angular_friction(self):
        return self._angular_friction

    @angular_friction.setter
    def angular_friction(self, value):
        self._set_param("angular_friction", value)

    @property
    def gravity(self):
        return self._gravity

    @gravity.setter
    def gravity(self, value):
        old = self._gravity
        self._gravity = value
        per_env = lambda g: isinstance(g, Tensor) and g.dim() == 2  # noqa: E731
        if not (per_env(old) and per_env(value) and old.shape == value.shape):
            self._touch()  # a new [B, 2] wind field is data, not structure: the plan stays valid

    @property
    def collision_filter(self):
        return self._collision_filter

    @collision_filter.setter
    def collision_filter(self, collision_filter: Callable[["Entity"], bool]):
        self._collision_filter = collision_filter
        self._touch()

    # lifecycle -------------------------------------------------------------------------
    def _spawn(self, dim_c: int, dim_p: int):
        self.state._spawn(dim_c, dim_p)

    def _reset(self, env_index):
        self.state._reset(env_index)

    def zero_grad(self):
        self.state.zero_grad()

    # state mutation protocol (ref core.py:733-761) ------------------------------------------
    def set_pos(self, pos: Tensor, batch_index):
        self._set_state_property("pos", pos, batch_index)

    def set_vel(self, vel: Tensor, batch_index):
        self._set_state_property("vel", vel, batch_index)

    def set_rot(self, rot: Tensor, batch_index):
        self._set_state_property("rot", rot, batch_index)

    def set_ang_vel(self, ang_vel: Tensor, batch_index):
        self._set_state_property("ang_vel", ang_vel, batch_index)

    def _set_state_property(self, name: str, new: Tensor, batch_index):
        assert (
            self.batch_dim is not None
        ), f"Tried to set property of {self.name} without adding it to the world"
        self._check_batch_index(batch_index)
        new = new.to(self.device)
        if batch_index is None:
            if new.dim() > 1 and new.shape[0] == self.batch_dim:
                setattr(self.state, name, new)
            else:
                setattr(self.state, name, new.repeat(self.batch_dim, 1))
        elif isinstance(batch_index, Tensor) and batch_index.dtype == torch.bool:
            # extension: a [B] bool mask selects the envs; `new` holds a row for every env (or
            # broadcasts), rows of unselected envs are ignored
            _write_rows(getattr(self.state, name), new, batch_index)
        else:
            getattr(self.state, name)[batch_index] = new
        self.notify_observers()

    def to(self, device: torch.device):
        TorchVectorizedObject.to(self, device)
        self.state.to(device)

    def render(self, env_index: int = 0):
        raise NotImplementedError("Rendering is outside the scope of the CUDA hot-path build")


class Landmark(Entity):
    def __init__(
        self,
        name: str,
        shape: Shape = None,
        movable: bool = False,
        rotatable: bool = False,
        collide: bool = True,
        density: float = 25.0,
        mass: float = 1.0,
        v_range: float = None,
        max_speed: float = None,
        color=Color.GRAY,
        is_joint: bool = False,
        drag: float = None,
        linear_friction: float = None,
        angular_friction: float = None,
        gravity: float = None,
        collision_filter: Callable[[Entity], bool] = lambda _: True,
    ):
        super().__init__(
            name,
            movable,
            rotatable,
            collide,
            density,
            mass,
            shape,
            v_range,
            max_speed,
            color,
            is_joint,
            drag,
            linear_friction,
            angular_friction,
            gravity,
            collision_filter,
        )


class Agent(Entity):
    def __init__(
        self,
        name: str,
        shape: Shape = None,
        movable: bool = True,
        rotatable: bool = True,
        collide: bool = True,
        density: float = 25.0,
        mass: float = 1.0,
        f_range: float = None,
        max_f: float = None,
        t_range: float = None,
        max_t: float = None,
        v_range: float = None,
        max_speed: float = None,
        color=Color.BLUE,
        alpha: float = 0.5,
        obs_range: float = None,
        obs_noise: float = None,
        u_noise: Union[float, Sequence[float]] = 0.0,
        u_range: Union[float, Sequence[float]] = 1.0,
        u_multiplier: Union[float, Sequence[float]] = 1.0,
        action_script: Callable[["Agent", "World"], None] = None,
        sensors: List = None,
        c_noise: float = 0.0,
        silent: bool = True,
        adversary: bool = False,
        drag: float = None,
        linear_friction: float = None,
        angular_friction: float = None,
        gravity: float = None,
        collision_filter: Callable[[Entity], bool] = lambda _: True,
        render_action: bool = False,
        dynamics: Dynamics = None,
        action_size: int = None,
        discrete_action_nvec: List[int] = None,
    ):
        super().__init__(
            name,
            movable,
            rotatable,
            collide,
            density,
            mass,
            shape,
            v_range,
            max_speed,
            color,
            is_joint=False,
            drag=drag,
            linear_friction=linear_friction,
            angular_friction=angular_friction,
            gravity=gravity,
            collision_filter=collision_filter,
        )
        if obs_range == 0.0:
            assert sensors is None, f"Blind agent cannot have sensors, got {sensors}"
        if action_size is not None and discrete_action_nvec is not None:
            if action_size != len(discrete_action_nvec):
                raise ValueError(
                    f"action_size {action_size} is inconsistent with discrete_action_nvec {discrete_action_nvec}"
                )
        if discrete_action_nvec is not None and not all(n > 1 for n in discrete_action_nvec):
            raise ValueError(
                f"All values in discrete_action_nvec must be greater than 1, got {discrete_action_nvec}"
            )

        self._obs_range = obs_range
        self._obs_noise = obs_noise
        self._f_range = f_range
        self._max_f = max_f
        self._t_range = t_range
        self._max_t = max_t
        self._action_script = action_script
        self._sensors = []
        if sensors is not None:
            for sensor in sensors:
                self.add_sensor(sensor)
        self._c_noise = c_noise
        self._silent = silent
        self._render_action = render_action
        self._adversary = adversary
        self._alpha = alpha

        self.dynamics = dynamics if dynamics is not None else Holonomic()
        if action_size is not None:
            self.action_size = action_size
        elif discrete_action_nvec is not None:
            self.action_size = len(discrete_action_nvec)
        else:
            self.action_size = self.dynamics.needed_action_size
        self.discrete_action_nvec = (
            [3] * self.action_size if discrete_action_nvec is None else discrete_action_nvec
        )
        self.dynamics.agent = self
        self._action = Action(
            u_range=u_range,
            u_multiplier=u_multiplier,
            u_noise=u_noise,
            action_size=self.action_size,
        )
        self._state = AgentState()

    def add_sensor(self, sensor):
        sensor.agent = self
        self._sensors.append(sensor)
        self._touch()

    @Entity.batch_dim.setter
    def batch_dim(self, batch_dim: int):
        Entity.batch_dim.fset(self, batch_dim)
        self._action.batch_dim = batch_dim

    @property
    def action_script(self):
        return self._action_script

    def action_callback(self, world: "World"):
        self._action_script(self, world)
        if self._silent or world.dim_c == 0:
            assert (
                self._action.c is None
            ), f"Agent {self.name} should not communicate but action script communicates"
        assert self._action.u is not None, f"Action script of {self.name} should set u action"
        assert (
            self._action.u.shape[1] == self.action_size
        ), f"Scripted action of agent {self.name} has wrong shape"
        if world.check_scripted_actions:
            # a device->host sync; World(check_scripted_actions=False) skips it
            assert (
                (self._action.u / self.action.u_multiplier_tensor).abs()
                <= self.action.u_range_tensor
            ).all(), f"Scripted physical action of {self.name} is out of range"

    @property
    def u_range(self):
        return self.action.u_range

    @property
    def obs_noise(self):
        return self._obs_noise if self._obs_noise is not None else 0

    @property
    def action(self) -> Action:
        return self._action

    @property
    def u_multiplier(self):
        return self.action.u_multiplier

    @property
    def max_f(self):
        return self._max_f

    @property
    def f_range(self):
        return self._f_range

    @property
    def max_t(self):
        return self._max_t

    @property
    def t_range(self):
        return self._t_range

    @property
    def silent(self):
        return self._silent

    @property
    def sensors(self):
        return self._sensors

    @property
    def u_noise(self):
        return self.action.u_noise

    @property
    def c_noise(self):
        return self._c_noise

    @property
    def adversary(self):
        return self._adversary

    def _spawn(self, dim_c: int, dim_p: int):
        if dim_c == 0:
            assert (
                self.silent
            ), f"Agent {self.name} must be silent when world has no communication"
        if self.silent:
            dim_c = 0
        super()._spawn(dim_c, dim_p)

    def _reset(self, env_index):
        self.action._reset(env_index)
        self.dynamics.reset(env_index)
        super()._reset(env_index)

    def zero_grad(self):
        self.action.zero_grad()
        self.dynamics.zero_grad()
        super().zero_grad()

    def to(self, device: torch.device):
        super().to(device)
        self.action.to(device)
        for sensor in self.sensors:
            sensor.to(device)


# ----------------------------------------------------------------------------------------
# World (ref core.py:1090-2919)
# ----------------------------------------------------------------------------------------
class World(TorchVectorizedObject):
    """Batched 2-D world whose ``step`` is one call into the CUDA physics kernels.

    Constructor arguments are the reference's (ref core.py:1091-1108).  Two extra keyword
    arguments exist only here: ``check_scripted_actions`` (keep the reference's range assert
    on scripted agents, which costs a host sync) and ``exact_broad_phase`` (reproduce the
    reference's batch-wide pair activation mask, ref core.py:2797-2801; on by default).
    """

    #: test seam: a callable ``world -> backend`` replacing the CUDA backend (used only by
    #: the CPU oracle in ``tests/`` and ``bench.py --impl reference``)
    _backend_factory = None

    def __init__(
        self,
        batch_dim: int,
        device: torch.device,
        dt: float = 0.1,
        substeps: int = 1,
        drag: float = DRAG,
        linear_friction: float = LINEAR_FRICTION,
        angular_friction: float = ANGULAR_FRICTION,
        x_semidim: float = None,
        y_semidim: float = None,
        dim_c: int = 0,
        collision_force: float = COLLISION_FORCE,
        joint_force: float = JOINT_FORCE,
        torque_constraint_force: float = TORQUE_CONSTRAINT_FORCE,
        contact_margin: float = 1e-3,
        gravity: Tuple[float, float] = (0.0, 0.0),
        check_scripted_actions: bool = True,
        exact_broad_phase: bool = True,
    ):
        assert batch_dim > 0, f"Batch dim must be greater than 0, got {batch_dim}"
        super().__init__(batch_dim, torch.device(device) if device is not None else None)
        self._agents: List[Agent] = []
        self._landmarks: List[Landmark] = []
        self._x_semidim = x_semidim
        self._y_semidim = y_semidim
        self._dim_p = 2
        self._dim_c = dim_c
        self._dt = dt
        self._substeps = substeps
        self._sub_dt = self._dt / self._substeps
        self._drag = drag
        self._gravity = torch.tensor(gravity, device=self.device, dtype=torch.float32)
        self._gravity_host = tuple(float(g) for g in gravity)
        self._linear_friction = linear_friction
        self._angular_friction = angular_friction
        self._collision_force = collision_force
        self._joint_force = joint_force
        self._contact_margin = contact_margin
        self._torque_constraint_force = torque_constraint_force
        self._joints = {}
        self._collidable_pairs = [
            {Sphere, Sphere},
            {Sphere, Box},
            {Sphere, Line},
            {Line, Line},
            {Line, Box},
            {Box, Box},
        ]
        self.entity_index_map = {}
        self.check_scripted_actions = check_scripted_actions
        self.exact_broad_phase = exact_broad_phase
        # compiled-plan bookkeeping
        self._slab: Optional[StateSlab] = None
        self._layout_version = 0
        self._slab_version = -1
        self._plan_version = 0
        self._backend = None
        self._factory_at_init = type(self)._backend_factory
        # device-side reset bookkeeping
        #: index of this world's env 0 in the whole job when ``batch_dim`` is one shard of a
        #: multi-GPU job (``shard.make_shard_env``): the respawn kernel numbers its random streams by
        #: global env, so a shard places entities exactly where the unsharded job would
        self.env_offset = 0
        self._reset_count: Optional[Tensor] = None
        self._spawn_status: Optional[Tensor] = None
        #: Philox key of the respawn kernel: set by Environment.seed() of the env that owns this world
        #: (None: torch.initial_seed() at call time, e.g. for a World used without an Environment)
        self.spawn_seed: Optional[int] = None
        self._spawn_calls = 0

    # -- construction -------------------------------------------------------------------
    def add_agent(self, agent: Agent):
        """Only way to add agents to the world"""
        agent.batch_dim = self._batch_dim
        agent.to(self._device)
        agent._spawn(dim_c=self._dim_c, dim_p=self.dim_p)
        agent._world = self
        self._agents.append(agent)
        self._layout_changed()

    def add_landmark(self, landmark: Landmark):
        """Only way to add landmarks to the world"""
        landmark.batch_dim = self._batch_dim
        landmark.to(self._device)
        landmark._spawn(dim_c=self.dim_c, dim_p=self.dim_p)
        landmark._world = self
        self._landmarks.append(landmark)
        self._layout_changed()

    def add_joint(self, joint):
        assert self._substeps > 1, "For joints, world substeps needs to be more than 1"
        if joint.landmark is not None:
            self.add_landmark(joint.landmark)
        for constraint in joint.joint_constraints:
            constraint._world = self
            self._joints[
                frozenset({constraint.entity_a.name, constraint.entity_b.name})
            ] = constraint
        self._invalidate_plan()

    def _layout_changed(self):
        self._layout_version += 1
        self._invalidate_plan()

    def _invalidate_plan(self):
        self._plan_version += 1

    def invalidate_plan(self):
        """Call after mutating a static physical attribute the setters do not cover."""
        self._invalidate_plan()

    # -- slab ---------------------------------------------------------------------------
    def _ensure_slab(self) -> StateSlab:
        if self._slab is None or self._slab_version != self._layout_version:
            entities = self.entities
            slab = StateSlab(self._batch_dim, self._device, entities, self._agents)
            slab.bind(entities, self._agents)
            self._slab = slab
            self._slab_version = self._layout_version
        return self._slab

    @property
    def slab(self) -> StateSlab:
        return self._ensure_slab()

    def _get_backend(self):
        if self._backend is None:
            factory = self._factory_at_init or type(self)._backend_factory
            if factory is not None:
                self._backend = factory(self)
            else:
                from ..backend import CudaBackend

                self._backend = CudaBackend(self)
        return self._backend

    # -- bulk operations ---------------------------------------------------------------------
    #: device-side reset (``vmas_b200_reset_state`` / ``vmas_b200_spawn_entities``) for CUDA worlds;
    #: ``VMAS_B200_DEVICE_RESET=0`` keeps the reference's torch formulation (same results for the
    #: state zeroing; the respawn then draws from torch's generator instead of the kernel's stream)
    device_reset_enabled = os.environ.get("VMAS_B200_DEVICE_RESET", "1") != "0"

    @property
    def uses_device_reset(self) -> bool:
        return (
            type(self).device_reset_enabled
            and self._factory_at_init is None
            and type(self)._backend_factory is None
            and torch.device(self._device).type == "cuda"
        )

    @property
    def reset_count(self) -> Tensor:
        """``[B]`` int32: how many times each env has been reset (its episode number); part of the
        respawn kernel's random-number counter."""
        if self._reset_count is None or self._reset_count.device.type != torch.device(self._device).type:
            self._reset_count = torch.zeros(self._batch_dim, dtype=torch.int32, device=self._device)
        return self._reset_count

    def reset(self, env_index):
        """Zero the state of every entity in the selected envs (ref core.py:1179-1181).

        ``env_index``: ``None`` (all envs), an int (the reference's ``reset_at``), or — an extension —
        a ``[B]`` bool tensor flagging the envs to reset, handled without a host sync.
        """
        self._spawn_calls = 0
        if self.uses_device_reset:
            self._ensure_slab()
            self._get_backend().reset_state(env_index, self.reset_count)
            # what Agent._reset does besides zeroing the slab rows: the action buffers, the
            # dynamics model's own state (e.g. Drone) and the communication state
            for a in self._agents:
                a.action._reset(env_index)
                a.dynamics.reset(env_index)
                if self._dim_c > 0 and a.state.c is not None:
                    _zero_rows(a.state.c, env_index)
            return
        for e in self.entities:
            e._reset(env_index)
        if isinstance(env_index, Tensor):
            self.reset_count.add_(env_index.to(torch.int32))
        elif env_index is None:
            self.reset_count.add_(1)
        else:
            self.reset_count[env_index] += 1

    def spawn_positions(
        self,
        entities,
        env_index,
        min_dist: float,
        x_bounds,
        y_bounds,
        occupied_positions: Optional[Tensor] = None,
        occupied_entities=(),
        want_positions: bool = False,
        max_tries: int = 1 << 16,
    ) -> Optional[Tensor]:
        """Device-side ``ScenarioUtils.spawn_entities_randomly`` (ref utils.py:241-319): places
        ``entities`` (``None`` entries: only draw a position) in the selected envs, each at least
        ``min_dist`` from the occupied points, the ``occupied_entities`` and the ones placed before
        it.  At most ``MAX_SPAWN`` positions per launch; longer lists are chained.

        The random stream is keyed by ``torch.initial_seed()`` (what ``Environment.seed`` sets), the
        env, its episode number (:attr:`reset_count`) and the position of the call within the reset.
        """
        assert self.uses_device_reset, "spawn_positions needs a CUDA world (device-side reset)"
        backend = self._get_backend()
        if self._spawn_status is None:
            self._spawn_status = torch.zeros(1, dtype=torch.int32, device=self._device)
        entities, occupied_entities = list(entities), list(occupied_entities)
        chunk_size = backend._native.MAX_SPAWN
        assert len(occupied_entities) <= chunk_size, f"at most {chunk_size} occupied entities per spawn call"
        outs = []
        for lo in range(0, len(entities), chunk_size):
            chunk = entities[lo : lo + chunk_size]
            out = backend.spawn(
                chunk,
                env_index,
                min_dist,
                x_bounds,
                y_bounds,
                seed=self.spawn_seed if self.spawn_seed is not None else torch.initial_seed(),
                stream_id=self._spawn_calls,
                reset_count=self.reset_count,
                status=self._spawn_status,
                occupied=occupied_positions,
                occupied_entities=occupied_entities,
                want_positions=want_positions or lo + chunk_size < len(entities),
                max_tries=max_tries,
            )
            self._spawn_calls += 1
            if out is not None:
                outs.append(out)
                if lo + chunk_size < len(entities):  # later chunks keep away from this one
                    occupied_positions = out if occupied_positions is None else torch.cat(
                        [occupied_positions.expand(out.shape[0], -1, -1), out], dim=1
                    )
        if not want_positions:
            return None
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)

    def spawn_failures(self) -> int:
        """Number of (env, call) pairs whose rejection sampling ran out of attempts so far (the
        reference would still be looping).  Reads a device counter: one host sync."""
        return 0 if self._spawn_status is None else int(self._spawn_status.item())

    def zero_grad(self):
        return

    # -- read-only views ---------------------------------------------------------------------
    @property
    def agents(self) -> List[Agent]:
        return self._agents

    @property
    def landmarks(self) -> List[Landmark]:
        return self._landmarks

    @property
    def x_semidim(self):
        return self._x_semidim

    @property
    def y_semidim(self):
        return self._y_semidim

    @property
    def dt(self):
        return self._dt

    @property
    def substeps(self):
        return self._substeps

    @property
    def dim_p(self):
        return self._dim_p

    @property
    def dim_c(self):
        return self._dim_c

    @property
    def joints(self):
        return self._joints.values()

    @property
    def entities(self) -> List[Entity]:
        return self._landmarks + self._agents

    @property
    def policy_agents(self) -> List[Agent]:
        return [a for a in self._agents if a.action_script is None]

    @property
    def scripted_agents(self) -> List[Agent]:
        return [a for a in self._agents if a.action_script is not None]

    # -- hot path ---------------------------------------------------------------------------------
    def step(self):
        """Advance every env by ``dt`` (``substeps`` fused force→integrate passes).

        Stands in for ref core.py:1972-2015.  All physics runs in the CUDA extension.
        """
        self._get_backend().step()
        if self._dim_c > 0:
            for agent in self._agents:
                if not agent.silent:
                    agent.state.c = agent.action.c

    def cast_rays(
        self,
        entity: Entity,
        angles: Tensor,
        max_range: float,
        entity_filter: Callable[[Entity], bool] = lambda _: False,
    ) -> Tensor:
        """Distances ``[B, R]`` along rays leaving ``entity`` at world angles ``angles [B, R]``
        (ref core.py:1662-1786)."""
        return self._get_backend().cast_rays(entity, angles, max_range, entity_filter)

    def cast_ray(
        self,
        entity: Entity,
        angles: Tensor,
        max_range: float,
        entity_filter: Callable[[Entity], bool] = lambda _: False,
    ) -> Tensor:
        """Single ray per env, ``angles [B]`` → ``[B]`` (ref core.py:1628-1660)."""
        assert entity.state.pos.dim() == 2 and angles.dim() == 1
        assert entity.state.pos.shape[0] == angles.shape[0]
        return self.cast_rays(entity, angles.unsqueeze(-1), max_range, entity_filter).squeeze(-1)

    # -- geometric queries (ref core.py:1788-1969, 2788-2803) ------------------------------------------
    def get_distance_from_point(self, entity: Entity, test_point_pos, env_index: int = None):
        self._check_batch_index(env_index)
        out = self._get_backend().distance_from_point(entity, test_point_pos)
        if env_index is not None:
            out = out[env_index]
        return out

    def get_distance(self, entity_a: Entity, entity_b: Entity, env_index: int = None):
        self._check_batch_index(env_index)
        return self._get_backend().pair_distance(entity_a, entity_b)

    def is_overlapping(self, entity_a: Entity, entity_b: Entity, env_index: int = None):
        self._check_batch_index(env_index)
        out = self._get_backend().pair_overlap(entity_a, entity_b)
        if env_index is not None:
            out = out[env_index]
        return out

    # -- batched variants (extensions of the reference API: one kernel launch for many queries) -----
    def measure_lidars(self, sensors) -> Tensor:
        """``[Q, B, R]`` ranges of several LIDARs (same ray count) in one launch; equals
        ``torch.stack([s.measure() for s in sensors])`` and updates their last measurement."""
        out = self._get_backend().lidar_measure_many(list(sensors))
        for q, s in enumerate(sensors):
            s._last_measurement = out[q]
        return out

    def observe(self, plan) -> Tensor:
        """The ``[rows, B, width]`` block of an :class:`observe.ObservationPlan` (one row per
        agent): state-slab terms in one launch, all LIDAR terms in one more."""
        return self._get_backend().observe(plan)

    def distance_shaping(self, pairs, factor: float, prev: Tensor):
        """The shaping-reward pattern for ``K`` entity pairs in one launch: returns ``(dist, rew)``
        (``[K, B]`` each) with ``dist = |pos_a - pos_b|`` and ``rew = prev - dist * factor``, and
        overwrites ``prev`` (fp32 ``[K, B]``) with ``dist * factor`` for the next step."""
        return self._get_backend().distance_shaping(list(pairs), float(factor), prev)

    def get_distances(self, pairs) -> Tensor:
        """``[K, B]``: ``get_distance(a, b)`` for every ``(a, b)`` in ``pairs``, one launch."""
        return self._get_backend().pair_query_many(list(pairs), 0)

    def are_overlapping(self, pairs) -> Tensor:
        """``[K, B]`` bool: ``is_overlapping(a, b)`` for every pair, one launch."""
        return self._get_backend().pair_query_many(list(pairs), 1)

    def get_center_distances(self, pairs) -> Tensor:
        """``[K, B]``: distance between the two entities' centres (what ``collides`` thresholds)."""
        return self._get_backend().pair_query_many(list(pairs), 2)

    def collide_gates(self, pairs) -> Tensor:
        """``[K]`` bool: ``collides(a, b)`` for every pair as device flags (no host sync)."""
        pairs = list(pairs)
        key = (self._plan_version,) + tuple((id(a), id(b)) for a, b in pairs)
        cached = self.__dict__.setdefault("_gate_consts", {}).get(key)
        if cached is None:  # constants live on the device: no per-step upload (CUDA-graph safe)
            static = torch.tensor([self.static_collides(a, b) for a, b in pairs], device=self.device)
            thr = torch.tensor(
                [a.shape.circumscribed_radius() + b.shape.circumscribed_radius() for a, b in pairs],
                dtype=torch.float32,
                device=self.device,
            ).unsqueeze(-1)
            self._gate_consts.clear()
            cached = self._gate_consts[key] = (static, thr)
        static, thr = cached
        return static & (self.get_center_distances(pairs) <= thr).any(dim=-1)

    def static_collides(self, a: Entity, b: Entity) -> bool:
        """The batch-independent predicates of ref ``World.collides`` (core.py:2788-2796)."""
        if (not a.collides(b)) or (not b.collides(a)) or a is b:
            return False
        if not a.movable and not a.rotatable and not b.movable and not b.rotatable:
            return False
        if {a.shape.__class__, b.shape.__class__} not in self._collidable_pairs:
            return False
        return True

    def collides(self, a: Entity, b: Entity) -> bool:
        """Reference semantics incl. the batch-wide overlap test (one device→host sync)."""
        if not self.static_collides(a, b):
            return False
        return bool(self.collides_tensor(a, b))

    def collides_tensor(self, a: Entity, b: Entity) -> Tensor:
        """``collides`` as a 0-dim bool tensor on the world's device: no host sync.

        True iff the static predicates hold and, in at least one env of the batch, the two
        circumscribed circles overlap (ref core.py:2797-2801).
        """
        if not self.static_collides(a, b):
            return torch.zeros((), dtype=torch.bool, device=self.device)
        thr = a.shape.circumscribed_radius() + b.shape.circumscribed_radius()
        d = torch.linalg.vector_norm(a.state.pos - b.state.pos, dim=-1)
        return (d <= thr).any()

    def to(self, device: torch.device):
        device = torch.device(device)
        super().to(device)
        for e in self.entities:
            e.to(device)
        self._slab = None
        self._slab_version = -1
        self._backend = None
        self._spawn_status = None  # device-resident scratch of the respawn kernel: re-created on the new device
        self._reset_count = None
        self._invalidate_plan()
